/*
 * auron_b200.h -- C ABI of libauron_b200.so, the H100-native drop-in for Apache Auron's native engine
 * (the Rust cdylib `libauron`).  Plain pointers and sizes only; batches cross the boundary through the
 * Arrow C Data Interface exactly as in the reference.
 *
 * Each entry point names the reference interface it replaces (paths relative to apache/auron):
 *
 *   auron_b200_call_native      <- Java_org_apache_auron_jni_JniBridge_callNative
 *                                  native-engine/auron/src/exec.rs:42-118 (+ rt.rs:75-248 start)
 *   auron_b200_schema           <- AuronCallNativeWrapper.importSchema upcall, rt.rs:167-170
 *   auron_b200_next_batch       <- Java_..._JniBridge_nextBatch, exec.rs:122-129 (+ rt.rs:250-280,
 *                                  importBatch upcall :258-262)
 *   auron_b200_finalize_native  <- Java_..._JniBridge_finalizeNative, exec.rs:133-140 (rt.rs:282-306)
 *   auron_b200_on_exit          <- Java_..._JniBridge_onExit, exec.rs:144-149
 *   auron_b200_metrics          <- update_metrics walk, native-engine/auron/src/metrics.rs:22-58
 *   auron_b200_metrics_walk     <- update_metric_node (tree-shaped walk), metrics.rs:22-50
 *   auron_callbacks             <- the JNI upcalls the engine makes on the hot path
 *                                  (native-engine/auron-jni-bridge/src/jni_bridge.rs:607-777,1485-1525)
 *
 * The JNI symbols themselves (same names/signatures as exec.rs) are exported by jni_face.cc on top of
 * these functions; see INTEGRATION.md.
 */
#ifndef AURON_B200_H
#define AURON_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

struct ArrowSchema;
struct ArrowArray;

typedef struct auron_shuffle_block {
    const char* path;      /* file segment: path + offset + length */
    int64_t offset;
    int64_t length;
    const uint8_t* data;   /* in-memory block: data + length (path == NULL) */
} auron_shuffle_block;

/* Upcalls (all optional except export_next_batch when the plan has an FFIReaderExec). */
typedef struct auron_callbacks {
    void* user;
    /* AuronArrowFFIExporter.exportNextBatch(long ptr) (ffi_reader_exec.rs:182-251): fill *out (an empty
     * ArrowArray owned by the engine, which will call out->release) with the next batch of the exporter
     * registered under resource_id.  Returns 1 = batch produced, 0 = end of input, <0 = error. */
    int (*export_next_batch)(void* user, const char* resource_id, struct ArrowArray* out);
    /* FSDataInputWrapper.readFully(pos, buf) through JniBridge.openFileAsDataInputWrapper
     * (scan/internal_file_reader.rs:64-68, parquet_exec.rs:294-397).  Returns bytes read or <0.
     * NULL => the engine reads `path` from the local file system. */
    int64_t (*read_fully)(void* user, const char* fs_resource_id, const char* path, int64_t pos, void* buf, int64_t len);
    /* JniBridge.isTaskRunning() (auron-jni-bridge/src/lib.rs:35-50).  NULL => always running. */
    int (*is_task_running)(void* user);
    /* Next shuffle block of the iterator registered under resource_id (IpcReaderExec: the Scala iterator of
     * AuronBlockObject, ipc_reader_exec.rs:186-207): a file segment (path, offset, length -- hasFileSegment) or an
     * in-memory buffer (data, length -- hasByteBuffer; must stay valid until the next call).  Returns 1 = block
     * produced, 0 = end of input, <0 = error.  Only needed when the plan has an IpcReaderExecNode. */
    int (*next_shuffle_block)(void* user, const char* resource_id, struct auron_shuffle_block* out);
    /* Non-zero: read_fully may be called from the engine's own reader threads, several at a time (the JNI face sets it:
     * its threads attach to the JVM like the reference's tokio workers do, and FSDataInputWrapper.readFully is
     * thread-safe).  Zero: every upcall is made on the thread that calls auron_b200_next_batch, one at a time, and the
     * scan neither prefetches nor splits reads. */
    int32_t upcalls_from_any_thread;
    /* JniBridge.{int,long,double,boolean,string}Conf(key) (auron-jni-bridge/src/conf.rs:20-116): the value of the
     * configuration entry `key` (the reference's names: "SPARK_IO_COMPRESSION_CODEC", "SPARK_IO_COMPRESSION_ZSTD_LEVEL",
     * ...) written to `value` as text, NUL-terminated.  Returns its length, or <0 when the host has no such entry (the
     * engine then falls back to its AURON_* environment variable, then to the reference's default).  May be NULL. */
    int (*get_conf)(void* user, const char* key, char* value, int32_t cap);
    /* IpcWriterExec (datafusion-ext-plans/src/ipc_writer_exec.rs:106-190): the consumer registered under resource_id -- a
     * Scala `ByteBuffer => Unit` on the JVM side (broadcast exchange: NativeBroadcastExchangeBase.scala:317-328) -- receives
     * the Auron compacted batch format, block by block (`u32 length | codec stream`, ipc_compression.rs:84-103).  `data` is
     * valid during the call only.  Returns 0, or <0 on error.  Only needed when the plan has an IpcWriterExecNode. */
    int (*write_ipc)(void* user, const char* resource_id, const uint8_t* data, int64_t len);
    /* AuronBlockObject.throwFetchFailed(errmsg) (ipc_reader_exec.rs:211-219): the shuffle data read through resource_id is
     * corrupt.  A Spark host turns this into a FetchFailedException, so that the map output is recomputed instead of the
     * task failing for good.  Called before the engine returns the error from next_batch.  May be NULL. */
    void (*fetch_failed)(void* user, const char* resource_id, const char* message);
} auron_callbacks;

typedef struct auron_task auron_task;

/* Decode a protobuf TaskDefinition (auron.proto:790-795), build the operator tree and start the task on
 * CUDA device `device`.  Returns NULL on failure (see auron_b200_last_error). */
auron_task* auron_b200_call_native(const uint8_t* task_definition, size_t len, const auron_callbacks* callbacks, int device);
/* Output schema of the task's root operator.  Caller releases *out.  0 = ok, <0 = error. */
int auron_b200_schema(auron_task* task, struct ArrowSchema* out);
/* Next output batch (a struct array, one child per column; move semantics, caller calls out->release).
 * 1 = batch delivered, 0 = end of stream, <0 = error. */
int auron_b200_next_batch(auron_task* task, struct ArrowArray* out);
/* Cancel outstanding work, free the task.  Safe before the stream is exhausted (rt.rs:282-298). */
void auron_b200_finalize_native(auron_task* task);
void auron_b200_on_exit(void);
/* Thread-local message of the last failing call on this thread. */
const char* auron_b200_last_error(void);

/* Walk the operator tree depth-first (same order as the JVM MetricNode tree) reporting (name, value). */
typedef void (*auron_metric_fn)(void* user, int depth, const char* operator_name, const char* metric_name, int64_t value);
int auron_b200_metrics(auron_task* task, auron_metric_fn fn, void* user);
/* The same walk with the tree shape made explicit, as update_metric_node needs it (metrics.rs:22-50: MetricNode.getChild(i)
 * per plan child): `enter` is called once per operator before its metrics, with its depth and its index among the
 * children of its parent; operators without metrics are still entered. */
typedef void (*auron_metric_node_fn)(void* user, int depth, int child_index, const char* operator_name);
int auron_b200_metrics_walk(auron_task* task, auron_metric_node_fn enter, auron_metric_fn fn, void* user);

/* ---- device-resident inputs (no counterpart in the reference: HBM residency for the GPU engine) ----
 * Copies `batch` to HBM and appends it to the resource `resource_id`; an FFIReaderExec whose
 * export_iter_provider_resource_id equals resource_id then streams the resident batches without any
 * host transfer.  The batch is NOT released by the call. */
int auron_b200_put_device_batch(const char* resource_id, const struct ArrowArray* batch, const struct ArrowSchema* schema, int device);
void auron_b200_drop_device_resource(const char* resource_id);
/* The HBM budget all spillable operators of this process share on `device` (aggregate tables, sorted runs): the analogue of the
 * executor-wide budget of auron-memmgr (native-engine/auron-memmgr/src/lib.rs:201-423, sized there from spark.auron.memoryFraction).
 * bytes <= 0 restores the default (40 % of the device memory, or AURON_HBM_BUDGET_BYTES).  Returns the budget now in force. */
int64_t auron_b200_set_hbm_budget(int device, int64_t bytes);
/* Same idea for Parquet: copies a whole file image to HBM under `path`; a ParquetScanExec whose
 * PartitionedFile.path equals `path` then decodes page payloads in place (no host transfer, no IO). */
int auron_b200_put_device_file(const char* path, const uint8_t* bytes, size_t len, int device);
void auron_b200_drop_device_file(const char* path);
/* Host-resident file image (the JVM side already holds the file in a direct / pinned buffer, e.g. a cached block):
 * the scan uploads the projected column chunks straight from `bytes` (cudaMemcpyAsync per chunk, no read_fully /
 * pread round trip).  `bytes` stays owned by the caller and must outlive every task that scans `path`; pinned
 * memory gives full PCIe rate, pageable memory works but is staged by the driver. */
int auron_b200_put_host_file(const char* path, const uint8_t* bytes, size_t len);
void auron_b200_drop_host_file(const char* path);

/* ---- in-box repartition over NVLink (no counterpart in the reference, which shuffles through Spark's block manager:
 * datafusion-ext-plans/src/shuffle/ and ipc_reader_exec.rs).  One process per GPU; rank 0 creates the id, the host
 * runtime distributes it, every rank calls init once.  A ShuffleWriterExecNode whose output_data_file is
 * "nccl://<name>" then performs hash partitioning + all-to-all-v and streams out the rows of the partitions this rank
 * owns (partition p -> rank p * world / partition_count). */
int auron_b200_nccl_unique_id(uint8_t out_id[128]);
int auron_b200_nccl_init(const uint8_t id[128], int rank, int world, int device);
void auron_b200_nccl_finalize(void);

/* ---- kernel-level entry points (one per device algorithm; used by tests, ncu captures, bench) ----
 * Inputs/outputs are host Arrow struct arrays; columns named by index. */
/* create_murmur3_hashes / create_xxhash64_hashes (datafusion-ext-commons/src/spark_hash.rs:28-57):
 * kind 0 = murmur3 -> int32 column, 1 = xxhash64 -> int64 column. */
int auron_b200_k_hash(const struct ArrowArray* batch, const struct ArrowSchema* schema, const int32_t* cols, int32_t ncols, int32_t kind,
                      int64_t seed, struct ArrowArray* out, struct ArrowSchema* out_schema, int device);
/* evaluate_partition_ids (datafusion-ext-plans/src/shuffle/mod.rs:163-188) -> int32 column */
int auron_b200_k_partition_ids(const struct ArrowArray* batch, const struct ArrowSchema* schema, const int32_t* cols, int32_t ncols,
                               int32_t num_partitions, struct ArrowArray* out, struct ArrowSchema* out_schema, int device);
/* Decodes a TaskDefinition exactly as auron_b200_call_native does (same planner) but on no device, and writes the resulting
 * operator tree as JSON: per operator its reference name (`ExecutionPlan::name()`), output schema, the attributes decoded from the
 * plan node (expressions as text, join type / sides / keys, aggregate functions and modes, sort keys, limit, partitioning, scan files
 * and projection, resource ids) and its children.  What PhysicalPlanner::create_plan (auron-planner/src/planner.rs:114-760) would
 * build, made inspectable.  Returns the JSON length (text truncated to cap - 1 bytes) or -1 (auron_b200_last_error).  Host only. */
int64_t auron_b200_explain(const uint8_t* task_definition, size_t len, char* out, int64_t cap);
/* UTC offset (seconds east) the engine's time-zone tables give for `zone` at `utc_second`: what the device looks up for the
 * date/time functions that take a session time zone (spark_dates.rs:93-110,200-227, chrono-tz in the reference).
 * Returns 0 and fills *offset, or -1 when `zone` is not an IANA zone name.  Host only: usable without a GPU. */
int auron_b200_tz_offset(const char* zone, int64_t utc_second, int32_t* offset);
/* Lowercase hex digest of `len` bytes, computed by the same compression and padding code the device's md5 / sha2 kernels run
 * (Spark_MD5, Spark_Sha224/256/384/512, spark_crypto.rs:33-105).  `alg` is the digest length in bits: 128 (MD5), 224, 256, 384
 * or 512.  Writes 32 / 56 / 64 / 96 / 128 characters to `out` (no terminator) and returns that count, or -1 for an unknown `alg`.
 * Host only: usable without a GPU. */
int auron_b200_digest_hex(int32_t alg, const uint8_t* bytes, int64_t len, char* out);
/* CAST(float AS STRING) of the float32 (bits 32) or float64 (bits 64) with bit pattern `value`, by the code the device's expression
 * VM runs: Java's Float / Double.toString as specified since JDK 19.  Writes at most 24 characters to `out` (no terminator) and
 * returns that count, or -1 for a bad argument.  Host only: usable without a GPU. */
int auron_b200_float_to_text(int32_t bits, uint64_t value, char* out);
/* CAST(text AS FLOAT / DOUBLE) of `len` bytes, Spark's non-ANSI semantics, by the code the device runs: writes the float32 (bits 32)
 * or float64 (bits 64) bit pattern to *value and returns 1, returns 0 where the cast gives NULL, -1 for a bad argument.
 * Host only: usable without a GPU. */
int auron_b200_text_to_float(int32_t bits, const uint8_t* text, int64_t len, uint64_t* value);
/* Decompress the ZSTD data in[0, in_len) (Zstandard and skippable frames back to back, a Parquet ZSTD page body) into out[0, out_len)
 * with the decoder the Parquet scan runs on the device.  Returns the bytes written, or -1 (auron_b200_last_error) when the data are
 * malformed or decode to more than out_len bytes.  Host only: usable without a GPU. */
int64_t auron_b200_zstd_decompress(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_len);
/* What the engine's Parquet metadata reader sees in the local file `path`, as JSON: footer (schema elements, row groups, column
 * chunks with codec / sizes / offsets / statistics as hex) plus, per chunk, the walk of its page headers (page counts, value
 * counts, encodings; SNAPPY bodies are run through the engine's block decoder).  The reference reads the same structures with
 * the `parquet` crate (parquet_exec.rs:175-197).  Returns the JSON length (the text is truncated to cap - 1 bytes), or -1 with the
 * error message in `out`.  Host only: usable without a GPU. */
int64_t auron_b200_parquet_describe(const char* path, char* out, int64_t cap);
/* number of kernels this library has launched in the calling process (bench.py "gpu_launches") */
int64_t auron_b200_kernel_launches(void);
/* micro-benchmark hook: runs `iters` launches of a named kernel over device-resident resource data and
 * returns the average milliseconds per launch measured with CUDA events on the launching stream. */
double auron_b200_time_kernel(const char* kernel, const char* resource_id, int32_t iters, int32_t arg0, int device);

#ifdef __cplusplus
}
#endif
#endif /* AURON_B200_H */
