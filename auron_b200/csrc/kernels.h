// kernels.h -- host-callable API of the kernel layer (one entry per device algorithm).
// All functions enqueue work on ctx.stream; those that return host-side counts synchronise.
#pragma once
#include "common.h"

namespace auron {

// ----------------------------------------------------------------------------- k_basic.cu
void launch_count(Ctx& ctx, int n = 1);
// exclusive prefix sums; in == out allowed.  If total != nullptr the grand total is written there (device).
void exclusive_scan_i32(Ctx& ctx, const int32_t* in, int32_t* out, int64_t n, int32_t* total_dev);
void exclusive_scan_i64(Ctx& ctx, const int64_t* in, int64_t* out, int64_t n, int64_t* total_dev);
// number of set bits among the first n bits (synchronises)
int64_t count_set_bits(Ctx& ctx, const uint8_t* bitmap, int64_t n);
// bitmap -> ascending row indices of set bits; returns count (synchronises)
Buf mask_to_indices(Ctx& ctx, const uint32_t* mask_words, int64_t n_rows, int64_t* count_out);
// dst bitmap (pre-zeroed) |= src bits [src_off, src_off+n) placed at dst_off
void copy_bits(Ctx& ctx, uint8_t* dst, int64_t dst_off, const uint8_t* src, int64_t src_off, int64_t n);
void fill_iota_i32(Ctx& ctx, int32_t* out, int64_t n, int32_t start);
// out[i] = a[i] & b[i] over whole words; either may be nullptr (treated as all ones); returns nullptr if both null
Buf and_bitmaps(Ctx& ctx, const uint8_t* a, const uint8_t* b, int64_t n_bits);
Buf not_bitmap(Ctx& ctx, const uint8_t* a, int64_t n_bits);

// gather: out[i] = in[idx[i]]; idx[i] < 0 yields NULL (outer joins).  idx == nullptr => identity copy.
ColumnPtr take(Ctx& ctx, const Column& in, const int32_t* idx, int64_t n_out, bool idx_may_be_negative);
BatchPtr take_batch(Ctx& ctx, const Batch& in, const int32_t* idx, int64_t n_out, bool idx_may_be_negative);
ColumnPtr concat_columns(Ctx& ctx, const std::vector<ColumnPtr>& cols);
BatchPtr concat_batches(Ctx& ctx, const std::vector<BatchPtr>& batches);
ColumnPtr slice_column(Ctx& ctx, const Column& in, int64_t off, int64_t len);
BatchPtr slice_batch(Ctx& ctx, const Batch& in, int64_t off, int64_t len);

// ----------------------------------------------------------------------------- k_list.cu
// Spark_StringSplit (spark_strings.rs:93-115): the pieces of each utf8 row between the leftmost non-overlapping matches of a
// non-empty pattern; a NULL row gives a NULL list
ColumnPtr string_split(Ctx& ctx, const Column& s, const std::string& pattern, const DType& out_type);
// Spark_MakeArray: row i = [args[0][i], ..., args[k-1][i]] (never NULL)
ColumnPtr make_array(Ctx& ctx, const std::vector<ColumnPtr>& args, int64_t n, const DType& out_type);
// the one list `elems` (NULL: is_null) in each of n rows
ColumnPtr broadcast_list(Ctx& ctx, const ColumnPtr& elems, bool is_null, int64_t n, const DType& out_type);
// explode / posexplode of a list column over n selected rows (row s of the list is input row sel[s]; sel == nullptr: s):
// rows_cum / bytes_cum = exclusive scans [n + 1] of the output rows per input row and of the bytes they copy of var_cols
constexpr int kMaxExplodeVarCols = 32;
void explode_scan(Ctx& ctx, const Column& list, bool outer, const std::vector<ColumnPtr>& var_cols, const int32_t* sel, int64_t n, Buf* rows_cum,
                  Buf* bytes_cum);
// end r1 of the piece that starts at selected row r0: the most rows within both limits, at least one (synchronises)
int64_t explode_cut(Ctx& ctx, const Buf& rows_cum, const Buf& bytes_cum, int64_t n, int64_t r0, int64_t max_rows, int64_t max_bytes, int64_t* out_rows,
                    int64_t* out_bytes);
// the n_out output rows of piece [r0, r1): input row, list element (-1 = the NULL row of outer) and, when pos != nullptr, the
// position (NULL in the outer row)
void explode_map(Ctx& ctx, const Column& list, const int32_t* sel, const Buf& rows_cum, int64_t r0, int64_t r1, int64_t n_out, int32_t* row_idx,
                 int32_t* elem_idx, int32_t* pos, uint32_t* pos_valid);

// ----------------------------------------------------------------------------- k_hash.cu
// Spark-compatible chained column hashing (spark_hash.rs:28-57). kind 0 murmur3 -> int32 out, 1 xxhash64 -> int64 out
Buf hash_columns(Ctx& ctx, const std::vector<ColumnPtr>& cols, int64_t n, int kind, int64_t seed);
// pmod(murmur3(cols, seed 42), num_parts)  (shuffle/mod.rs:163-188) -> int32[n]
Buf murmur3_partition_ids(Ctx& ctx, const std::vector<ColumnPtr>& cols, int64_t n, int32_t num_parts, int32_t seed = 42);
Buf bound_ranks(Ctx& ctx, const int32_t* perm, int64_t n, int64_t nb);   // range partitioning (k_sort.cu)
Buf round_robin_partition_ids(Ctx& ctx, int64_t n, int64_t start, int32_t num_parts);   // (i + start) % num_parts

// ----------------------------------------------------------------------------- k_digest.cu
// Spark md5 / sha2 as lowercase hex (spark_crypto.rs:33-105); the algorithm is named by its digest length in bits
enum DigestAlg : int { DIGEST_MD5 = 128, DIGEST_SHA224 = 224, DIGEST_SHA256 = 256, DIGEST_SHA384 = 384, DIGEST_SHA512 = 512 };
int digest_hex_width(int alg);   // 32 / 56 / 64 / 96 / 128 characters, -1 for an unknown algorithm
// lens[i] = hex width when row sel[i] (sel == nullptr: row i) of in_valid is valid, else 0; out_valid = that validity
void digest_lengths(Ctx& ctx, const uint8_t* in_valid, const int32_t* sel, int64_t n, int alg, uint32_t* out_valid, int64_t* lens);
// hex digests of the utf8 / binary rows sel[i] into out at out_off[i]; an empty output range marks a NULL row
void digest_hex(Ctx& ctx, int alg, const int32_t* in_off, const uint8_t* in_data, const int32_t* sel, int64_t n, const int32_t* out_off,
                uint8_t* out);
// the same computation on the CPU: writes digest_hex_width(alg) characters to out, returns that width or -1
int digest_hex_host(int alg, const uint8_t* bytes, int64_t len, char* out);

// ----------------------------------------------------------------------------- k_expr.cu: the float <-> text casts on the CPU
// (float_text.cuh, the code the device runs).  bits: 32 or 64; values are bit patterns.
int float_to_text_host(int bits, uint64_t value, char* out);   // Java's Float / Double.toString into out (>= 24 bytes); the length
bool text_to_float_host(int bits, const uint8_t* text, int32_t len, uint64_t* value);   // Spark's CAST; false: NULL
// k_zstd.cu: the device's ZSTD page decoder (zstd_dec.cuh) on the CPU; bytes written into out[0, out_len), or -1 (malformed or too long)
int64_t zstd_decompress_host(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_len);

// ----------------------------------------------------------------------------- k_rowkeys.cu
// Row-key view over key columns for hash aggregation / joins (general path)
struct KeyColDesc {
    const void* data;
    const uint8_t* validity;
    const int32_t* offsets;
    int32_t type;   // TypeId
    int32_t width;  // bytes (0 => bool bitmap / varlen)
};
constexpr int kMaxKeyCols = 8;
struct RowKeys {
    KeyColDesc c[kMaxKeyCols];
    int32_t ncols;
};
RowKeys make_row_keys(const std::vector<ColumnPtr>& cols);

// ----------------------------------------------------------------------------- k_agg.cu
enum AccKind : int32_t {
    ACC_SUM_I64 = 0,   // in: int64-extended ints (i8..i64) -> acc int64
    ACC_SUM_F64 = 1,   // in: f32/f64 -> acc f64
    ACC_SUM_DEC = 2,   // in: decimal128 -> acc decimal128 (wrapping i128)
    ACC_COUNT = 3,     // +1 when all args valid (up to 4 arg validities) ; acc int64
    ACC_ADD_I64 = 4,   // merge of COUNT: acc += value
    ACC_MIN = 5,       // by input type
    ACC_MAX = 6,
    ACC_FIRST = 7,     // value of the smallest row index (+ is_set)
    ACC_FIRST_IGNORES_NULL = 8,
    ACC_MIN_STR = 9,   // utf8 / binary input: the accumulator holds the ROW of the current extreme (byte-wise order), -1 = none
    ACC_MAX_STR = 10,
};
struct AccSpec {
    AccKind kind;
    ColumnPtr input;                  // may be null for COUNT(*) style (no args)
    std::vector<ColumnPtr> extra;     // extra args for COUNT(a,b,..) validity; FIRST merge: is_set column
    DType out_type;                   // accumulator column type
    ColumnPtr gather_from;            // FIRST merge: column the winning position is gathered from (default: input)
    int input_id = -1;                // producers without input columns (fused scan): identifies the source column, so that
                                      // SUM(x) pairs with COUNT(x) for its validity
};
struct GroupedResult {
    BatchPtr keys;                    // distinct key columns (dense groups)
    std::vector<ColumnPtr> accs;      // one column per AccSpec (FIRST adds a second bool column after it)
    int64_t num_groups = 0;
};
// Hash-aggregate one device-resident batch.  sel (optional) = row selection (filter fused into the aggregate).
// fast_key_out (optional, single fixed-width integer key only): emit the group key in this wider integer type.
GroupedResult hash_aggregate(Ctx& ctx, const std::vector<ColumnPtr>& keys, const std::vector<AccSpec>& accs,
                             const int32_t* sel, int64_t n_rows, const DType* fast_key_out = nullptr,
                             const uint32_t* selmask = nullptr, int64_t n_selected = -1);   // selmask: pending filter bit mask (see k_agg.cu)
// ---- persistent direct-address aggregate table (single integer key with a small value range)
struct DirectAgg;
constexpr int kDirectMaxAccs = 16;
struct DirectAggView {            // device pointers a producer kernel updates: slot = key - kmin, slot `range` = NULL key
    int32_t n;
    int32_t kind[kDirectMaxAccs];                 // AccKind
    unsigned long long* acc[kDirectMaxAccs];      // [range + 1]
    uint8_t* valid[kDirectMaxAccs];               // [range + 1] "accumulator holds a value" flags, or nullptr (COUNT; SUM paired with a COUNT)
    uint8_t* seen;                                // [range + 1] group exists although no accumulator shows it
    int32_t* oor;                                 // set to 1 by a producer that meets a key outside the range
    long long kmin;
    int64_t range;
};
std::shared_ptr<DirectAgg> direct_agg_create(Ctx& ctx, const std::vector<AccSpec>& specs, long long kmin, long long kmax);   // kmin > kmax: empty range
DirectAggView direct_agg_view(const DirectAgg& da);
void direct_agg_grow(Ctx& ctx, DirectAgg& da, long long kmin, long long kmax);   // widen to cover [kmin, kmax] as well (rebases the table)
bool direct_agg_out_of_range(Ctx& ctx, const DirectAgg& da);                      // synchronises
int64_t direct_agg_span_limit();
GroupedResult direct_agg_finish(Ctx& ctx, DirectAgg& da, const DType& key_type, bool key_nullable, const int32_t* sel = nullptr);
// no grouping keys: one output row
std::vector<ColumnPtr> global_aggregate(Ctx& ctx, const std::vector<AccSpec>& accs, const int32_t* sel, int64_t n_rows,
                                        const uint32_t* selmask = nullptr);
// AVG final merge (agg/avg.rs:151-179)
ColumnPtr avg_finalize(Ctx& ctx, const Column& sum, const Column& cnt, const DType& out_type);

// ----------------------------------------------------------------------------- k_join.cu
struct JoinTable;   // opaque device hash table over build keys
std::shared_ptr<JoinTable> join_build(Ctx& ctx, const std::vector<ColumnPtr>& build_keys, int64_t n_build);
bool join_table_has_null_key(const JoinTable& t);
bool join_table_unique_fast(const JoinTable& t);   // no duplicate build keys, single fixed-width key
// probe of such a table: partner build row per probe row (-1 = none) + match mask; returns the number of matches
int64_t join_probe_unique(Ctx& ctx, const JoinTable& t, const ColumnPtr& probe_key, int64_t n_probe, Buf* build_idx, Buf* mask);
struct JoinPairs {
    Buf probe_idx, build_idx;   // int32 each; -1 = no partner (outer)
    int64_t count = 0;
};
// inner pairs (+ unmatched probe rows as (i,-1) when probe_outer).  matched_build (bitmap over build rows,
// pre-zeroed, may be null) receives matched flags.  probe_matched_out (optional) = bitmap over probe rows.
JoinPairs join_probe(Ctx& ctx, const JoinTable& t, const std::vector<ColumnPtr>& probe_keys, int64_t n_probe, bool probe_outer,
                     uint32_t* matched_build, Buf* probe_matched_out);

// ----------------------------------------------------------------------------- k_window.cu
// rows sorted by (partition keys, order keys): flags[i] = 1 where row i starts a new group of `keys` (`also`: boundaries to inherit).
// prev: the keys of the previous batch's last row (one row per column; empty without keys) -- row 0 starts a group where they differ;
// nullptr: there is no previous row, row 0 starts a group.
Buf window_boundaries(Ctx& ctx, const std::vector<ColumnPtr>& keys, int64_t n, const uint8_t* also, const std::vector<ColumnPtr>* prev);
// the last row that starts a new group of `keys`, -1 when none does; row 0 counts only when prev (the keys of the row before it, one
// row per column) is given and differs.  Synchronises.
int64_t window_last_boundary(Ctx& ctx, const std::vector<ColumnPtr>& keys, int64_t n, const std::vector<ColumnPtr>* prev);
// the state of a running window function at the last row computed so far, carried into the next batch (empty: nothing before it)
struct WinCarry {
    Buf a, b;          // scan values at that row (see the functions below)
    ColumnPtr value;   // one-row column that owns its bytes (string MIN / MAX, NTH_VALUE)
};
// carry (optional): read when set, then replaced by the state at row n - 1
ColumnPtr window_rank_column(Ctx& ctx, int func /* 0 ROW_NUMBER, 1 RANK, 2 DENSE_RANK */, const uint8_t* pflags, const uint8_t* oflags, int64_t n, WinCarry* carry);
ColumnPtr window_agg_column(Ctx& ctx, int fn /* AggFunction: 0 MIN, 1 MAX, 2 SUM, 3 AVG, 4 COUNT */, const ColumnPtr& arg, const DType& out_type, const uint8_t* pflags, int64_t n,
                            WinCarry* carry);
ColumnPtr window_nth_column(Ctx& ctx, const ColumnPtr& values, int64_t nth, bool ignore_nulls, const uint8_t* pflags, int64_t n, WinCarry* carry);
// these look at the whole partition: the rows passed in hold complete partitions
ColumnPtr window_dist_column(Ctx& ctx, int func /* 6 PERCENT_RANK, 7 CUME_DIST */, const uint8_t* pflags, const uint8_t* oflags, int64_t n);
ColumnPtr window_lead_column(Ctx& ctx, const ColumnPtr& values, const ColumnPtr& defaults, int64_t offset, const uint8_t* pflags, int64_t n);
Buf window_le_mask(Ctx& ctx, const ColumnPtr& rank_col, int32_t k);   // bit mask of rows with rank <= k (WindowGroupLimit)

// ----------------------------------------------------------------------------- k_sort.cu
struct SortKeySpec {
    ColumnPtr col;
    bool asc = true;
    bool nulls_first = true;
};
// returns permutation (int32 row indices) that orders rows by keys (stable)
Buf sort_indices(Ctx& ctx, const std::vector<SortKeySpec>& keys, int64_t n_rows);
// external sort: normalised key words (most significant first) of the rows of a batch in row order -- comparable across batches;
// false when a key column is variable-length.  Samples / lower bounds over the words of a SORTED batch.
bool sort_key_words(Ctx& ctx, const std::vector<SortKeySpec>& keys, int64_t n, std::vector<Buf>* words);
std::vector<uint64_t> sample_sorted_words(Ctx& ctx, const std::vector<Buf>& words, int64_t n, int S);   // [S][W]
std::vector<int64_t> lower_bound_sorted_words(Ctx& ctx, const std::vector<Buf>& words, int64_t n, const std::vector<uint64_t>& splitters, int S);
// stable LSD radix sort of (u64 key, i32 value) pairs, in place over ping-pong buffers; bits [begin_bit, end_bit)
void radix_sort_pairs_u64(Ctx& ctx, Buf& keys, Buf& vals, int64_t n, int begin_bit, int end_bit);
// stable counting partition of rows by partition id: returns row order + offsets[num_parts+1] (device int64)
void partition_rows(Ctx& ctx, const int32_t* part_ids, int64_t n, int32_t num_parts, Buf* rows_out, Buf* offsets_out);

// ----------------------------------------------------------------------------- k_serde.cu
// Auron compacted batch format (batch_serde.rs:68-147): serialize rows [row_begin,row_end) of each partition
// segment into one device byte buffer; returns per-partition byte offsets (host) and the device buffer.
struct SerializedParts {
    Buf bytes;
    std::vector<int64_t> part_offsets;   // num_parts+1 (uncompressed payload offsets)
};
SerializedParts serialize_partitions(Ctx& ctx, const Batch& sorted_batch, const std::vector<int64_t>& row_offsets);
// LZ4-frame compression on device (k_lz4.cu): one warp per <= 64 KB block, then assembly of the partition streams
struct Lz4Block {
    const uint8_t* src;   // raw bytes of the block
    uint8_t* dst;         // scratch slot of lz4_block_bound(len) bytes
    int32_t len;
    int32_t pad;
};
struct Lz4Place {
    const uint8_t* src;   // compressed bytes (scratch) or the raw bytes when the block is stored
    uint8_t* dst;         // position of the block's 4-byte size word in the output image
    int32_t len;          // data bytes that follow the size word
    uint32_t size_word;   // len, high bit set for a stored block
    uint32_t flags;       // 1 = first block of its stream (writes u32 stream length + 7-byte frame header at dst-11), 2 = last (end mark)
    uint32_t stream_len;  // frame bytes of the stream (flag 1)
    uint8_t header[8];    // frame header (flag 1)
};
constexpr int kLz4BlockBytes = 64 * 1024;
inline int64_t lz4_block_bound(int64_t n) { return n + n / 255 + 32; }
void lz4_compress_blocks(Ctx& ctx, const Lz4Block* dev_blocks, int n_blocks, int32_t* dev_sizes);
void lz4_assemble(Ctx& ctx, const Lz4Place* dev_places, int n);
struct Lz4DBlock {          // one block of an LZ4 frame to decode (IpcReaderExec)
    const uint8_t* src;     // block data (after its 4-byte size word)
    uint8_t* dst;           // slot of dst_cap bytes in the payload buffer
    int32_t src_len, dst_cap;
    int32_t stored;         // 1 = the block is stored uncompressed
    int32_t pad;
};
void lz4_decompress_blocks(Ctx& ctx, const Lz4DBlock* dev_blocks, int n_blocks, int32_t* dev_sizes);   // sizes: decoded bytes, -1 = malformed

// read side (IpcReaderExec): one DeserSeg per batch of the column, offsets into the decompressed payload on the device
struct DeserSeg {
    int64_t validity_off;   // -1: no validity section (all rows valid)
    int64_t values_off;     // fixed: byte planes ; bool: bits ; utf8: four length planes
    int64_t out_row0;       // first output row of this batch
    int64_t n;
};
struct DeserCopy {          // utf8 payload bytes of one batch (or a piece of it)
    int64_t src, dst, len;
};
// device-side layout walk (payload decompressed on the GPU)
struct LayoutStream {
    int64_t begin, end;     // byte range of one codec stream's payload
};
struct LayoutSchema {
    int32_t ncols;
    uint8_t kind[64];       // 0 null, 1 bool, 2 fixed width, 3 utf8 / binary
    uint8_t width[64];
};
void deserialize_layout(Ctx& ctx, const uint8_t* dev_payload, const LayoutStream* dev_streams, int n_streams, const LayoutSchema& sch, const int32_t* dev_seg_base,
                        DeserSeg* dev_segs, int64_t* dev_sbytes, int64_t* dev_batch_rows, int32_t* dev_counts, int32_t* dev_flags);
ColumnPtr deserialize_column(Ctx& ctx, const DType& type, const uint8_t* dev_payload, const std::vector<DeserSeg>& segs, int64_t total_rows,
                             const std::vector<DeserCopy>& byte_copies, int64_t total_bytes);

}  // namespace auron
