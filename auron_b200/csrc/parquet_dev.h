// parquet_dev.h -- descriptors shared by the Parquet host walker (scan_parquet.cc) and the decode kernels.
#pragma once
#include "common.h"

namespace auron {

struct PqPage {
    const uint8_t* def_ptr;   // definition-level section (hybrid RLE, bit width 1), nullptr if none
    const uint8_t* val_ptr;   // value section (dictionary pages: bit-width byte + hybrid indices ; PLAIN: values)
    int32_t def_len, val_len;   // def_len == -1: v1 page decompressed on device, sections not split yet (pq_fix_v1_pages)
    int32_t num_values;       // rows of the page (flat columns)
    int32_t row_start;        // first output row of the page within the batch
    int32_t encoding;         // parquet Encoding of the values
    int32_t dict_id;          // index into PqColumnArgs::dicts
    int32_t all_null;
    int32_t plain_value_base; // strings: position of this page's first PLAIN value in the chunk value table
    int32_t job;              // v1 page decompressed on the device: index of its PqDecompJob / PqDecompResult, else -1
    int32_t delta_dst16;      // DELTA_BINARY_PACKED page: 1 + (offset / 16) of its PLAIN transcription in the batch's scratch buffer
                              // (pq_delta_to_plain rewrites val_ptr / val_len; `encoding` already says PLAIN), 0 = none
};
struct PqDict {
    const uint8_t* data;      // PLAIN-encoded fixed-width dictionary values
    int32_t num_values;
    int32_t value_base;       // strings: position of entry 0 in the value table
};
enum { PQ_MODE_VALUES = 0, PQ_MODE_INDEX = 1 };
// How one physical value becomes one value of the table's type, decided once per column on the host (scan_parquet.cc,
// conversion_of: the table of DESIGN section 4, "Parquet column conversions")
enum PqConv {
    PQ_CV_COPY = 0,     // the value as it is, stored at the output's width (also INT96 -> timestamp, booleans, byte arrays)
    PQ_CV_SEXT = 1,     // a signed INT32 / INT64 sign-extended to a wider integer, or to decimal128 as a value copy
                        //   (scan/mod.rs:131-136; also a decimal read at its own scale)
    PQ_CV_ZEXT = 2,     // an unsigned INT32 (UINT 8 / 16 / 32) zero-extended to a wider signed integer
    PQ_CV_I32_F64 = 3,  // a signed INT32 as the float64 of the same value
    PQ_CV_F32_F64 = 4,  // FLOAT widened to float64
    PQ_CV_TS_MUL = 5,   // INT64 timestamp x conv_mul into a finer unit; NULL when the product leaves int64
    PQ_CV_TS_DIV = 6,   // INT64 timestamp / conv_mul into a coarser unit, truncating toward zero
    PQ_CV_DEC = 7,      // a decimal on INT32 / INT64 / FLBA x (conv_mul_hi:conv_mul) > 1 into decimal128 (exact: the target is wide enough)
};
struct PqColumnArgs {
    const PqPage* pages;
    const PqDict* dicts;
    int32_t n_pages;
    int32_t phys_type, phys_width, type_length;
    int32_t out_type, out_width;
    int32_t max_def;
    int32_t mode;
    int32_t out_unit;   // T_TIMESTAMP output: 0 s, 1 ms, 2 us, 3 ns (INT96 pages are converted to it)
    int32_t conv;       // PqConv
    uint64_t conv_mul, conv_mul_hi;
    void* out;
    uint32_t* out_valid;
    int32_t* out_idx;
};
struct PqByteSection {
    const uint8_t* ptr;
    int64_t len;
    int32_t num_values;
    int32_t value_base;
};

// page decompression on device (k_snappy.cu): one warp per job
struct PqDecompJob {
    const uint8_t* src;
    uint8_t* dst;
    int32_t src_len, dst_len;
    int32_t kind;       // 0 = stored bytes, 1 = Snappy raw block, 2 = the front elements of a Snappy raw block (the preamble
                        //     counts the whole block; the job ends after src_len bytes, which decode to dst_len bytes),
                        //     3 = ZSTD frames, 4 = LZ4 raw block (PqJobKind)
    int32_t v1_levels;  // 1 = body of a nullable v1 data page ([u32 length][levels][values]): a final literal that holds the
                        //     whole value section is NOT copied, the page then reads its values from the compressed buffer
};
struct PqDecompResult {
    const uint8_t* tail_src;   // where the value section lives inside the compressed buffer
    int32_t tail_start;        // its offset in the uncompressed body, -1 = everything was copied
    int32_t pad;
};
struct PqDecompOut {
    Buf status;    // int32: 0 = ok, else 1 + index of the first failing job
    Buf results;   // PqDecompResult per job
};
enum PqJobKind { PQ_JOB_STORED = 0, PQ_JOB_SNAPPY = 1, PQ_JOB_SNAPPY_HEAD = 2, PQ_JOB_ZSTD = 3, PQ_JOB_LZ4 = 4 };
// jobs[0, n_snappy) are stored / Snappy jobs (k_snappy.cu), jobs[n_snappy, size) stored / ZSTD / LZ4_RAW jobs (k_zstd.cu)
PqDecompOut pq_decompress(Ctx& ctx, const std::vector<PqDecompJob>& jobs, size_t n_snappy);
void pq_decompress_zstd_lz4(Ctx& ctx, const std::vector<PqDecompJob>& jobs, size_t first, const PqDecompJob* dev_jobs, int32_t* status,
                            PqDecompResult* results);
// pages with def_len == -1: level / value sections from the body's length word (+ in-place value sections, see above)
void pq_fix_v1_pages(Ctx& ctx, PqPage* pages, int n, const PqDecompResult* results);
// pages with delta_dst16 != 0: DELTA_BINARY_PACKED values (width 4 or 8 bytes) -> PLAIN values at scratch + 16 (delta_dst16 - 1);
// status (int32, may be the decompression status word) is set to 0x40000000 + page when a stream is malformed
void pq_delta_to_plain(Ctx& ctx, PqPage* pages, int n, uint8_t* scratch, int width, int32_t* status);

// ---- one-level LIST columns (k_parquet_levels.cu).  The element values of a list page are contiguous and decode with the page
// decoders above as a required column; the level streams of the pages give the list layout.
struct PqLevelPage {
    const uint8_t* rep;       // repetition levels (hybrid RLE / bit-packed)
    const uint8_t* def;       // definition levels
    int32_t rep_len, def_len;
    int32_t n_slots;          // level slots of the page (its num_values: elements, empty lists and NULL lists)
    int32_t slot_start;       // first slot of the page within the batch's column
};
struct PqListShape {
    int32_t rep_bw, def_bw;   // bit widths of max_rep (1) and max_def
    int32_t list_def;         // def < list_def: a NULL list (0: the list is required)
    int32_t elem_def;         // list_def <= def < elem_def: an empty list; def >= elem_def: an element
    int32_t max_def;          // an element is NULL unless def == max_def
};
// Level pass over the n_slots slots of a batch's list column: offsets[0, n_rows] (row r owns elements [offsets[r], offsets[r + 1])),
// validity (n_rows bits, zeroed by the caller; nullptr when list_def == 0) and elem_idx[e] = index of element e's value among the
// non-null values, -1 for a NULL element.  counts (device, int64[4]): rows found, elements, non-null values, status (0 = ok, else
// 1 + a page whose levels are malformed).  Rows past n_rows are counted, never written.
void pq_list_levels(Ctx& ctx, const PqLevelPage* pages, int n_pages, int64_t n_slots, int64_t n_rows, const PqListShape& s, int32_t* offsets,
                    uint32_t* validity, int32_t* elem_idx, int64_t* counts);
// idx[e] = idx[e] < 0 ? -1 : value_idx[idx[e]] for e < n, in place (a list of strings: element -> value-table entry, one byte gather)
void pq_compose_index(Ctx& ctx, int32_t* idx, const int32_t* value_idx, int64_t n);

// scout + decode of one column; or in three steps, so that one scout launch serves every column of a batch
void pq_decode_pages(Ctx& ctx, const PqColumnArgs& a, const std::vector<PqPage>& host_pages);
struct PqPrepared {
    PqColumnArgs a;
    int n_tiles = 0;
    Buf tile_base, tiles, tile_valid;
};
PqPrepared pq_prepare(Ctx& ctx, const PqColumnArgs& a, const std::vector<PqPage>& host_pages);
void pq_scout_many(Ctx& ctx, const std::vector<PqPrepared*>& cols);
void pq_decode_prepared(Ctx& ctx, const PqPrepared& pr);
ColumnPtr pq_build_value_table(Ctx& ctx, const std::vector<PqByteSection>& secs, int64_t total_values, const DType& type);

// ---- fused ParquetScan -> Filter -> HashAggregate (k_fused.cu) -------------------------------------------------------
// The three operators of BASELINE config 2 run as ONE pass over the encoded pages: row tiles of FZ_TILE rows are unpacked
// into shared memory, the filter's per-column intervals are tested, and the selected rows update the direct-address
// accumulators -- the decoded Arrow columns are never written to HBM (parquet_exec.rs:151-204 -> filter_exec.rs:200-224 ->
// agg/agg_table.rs:99-135 as one kernel).  Pages of different columns need not line up: the scout cuts every page at the
// global-row multiples of FZ_TILE ("segments"), so a tile of any column is a short list of segments.
constexpr int FZ_TILE = 1024;
constexpr int FZ_MAX_COLS = 8;    // role-columns (a column used as predicate and as key counts twice)
constexpr int FZ_MAX_ACCS = 6;
// checkpoint of an RLE / bit-packed hybrid stream (offsets relative to the stream's first byte)
struct HybridCk {
    int32_t p_off, run_remaining, bp_base_off, bp_consumed;
    uint32_t rle_value;
    int32_t is_rle;
};
struct FzSeg {                    // rows [row0, row0 + n) of one page, all inside one global tile; self-contained (96 bytes) so
                                  // that the fused kernel reaches the page bytes with ONE dependent load per column
    int32_t page, row0, n, nvalid;   // nvalid: non-null values among them
    int64_t v0;                      // non-null values of the page before row0
    HybridCk idx;                    // dictionary-index stream at the segment's first value
    const uint8_t* vals;             // the page's value section (dictionary pages: its bit-width byte)
    const uint8_t* ddata;            // dictionary pages: PLAIN values of the dictionary
    int32_t val_len, bw;             // bw = bit width of the indices, -1 = PLAIN page
    int32_t ndict, dict_id;
    int64_t pad[2];                  // pad[0] bit 0: the index stream is "regular" (only full 63-group bit-packed runs before a last shorter
                                     // one, each behind a one-byte header), or the page is PLAIN: value k sits at an arithmetic position
};
static_assert(sizeof(FzSeg) == 96, "FzSeg is read with 16-byte vector loads");
struct FzScoutCol {               // one physical column to scout
    const PqPage* pages;
    const PqDict* dicts;
    int32_t n_pages, max_def;
    const int32_t* seg_base;      // [n_pages + 1] first segment of every page
    FzSeg* segs;
    int32_t* first_seg;           // [n_tiles] segment that starts global tile T
    uint32_t* valid;              // batch-wide validity bitmap (zeroed; nullptr when max_def == 0)
};
enum { FZ_PRED = 0, FZ_KEY = 1, FZ_VALUE = 2 };
struct FzColumn {                 // one role-column of the fused kernel
    const PqPage* pages;
    const PqDict* dicts;
    const FzSeg* segs;
    const int32_t* first_seg;
    const uint32_t* valid;
    int32_t role;
    int32_t stage_cap;            // bytes of shared memory one tile of this column may occupy in the TMA-staged kernel (0 = never staged)
    int64_t lo, hi;               // FZ_PRED: closed interval the value must lie in (NULL never passes)
    const uint32_t* pass_bits;    // FZ_PRED: the interval test evaluated on every dictionary entry, one bit each
    const int32_t* pass_off;      //          [n_dicts] first word of each dictionary in pass_bits
    const int32_t* dslot_base;    // FZ_KEY : [n_dicts] first slot of each dictionary in the dictionary-space accumulators
};
struct FzAcc {
    int32_t kind;                 // AccKind: ACC_SUM_I64, ACC_COUNT, ACC_MIN, ACC_MAX
    int32_t col;                  // role-column holding the argument, -1 = COUNT(*)
    unsigned long long* direct;   // [range + 1] accumulators addressed by key - kmin (slot `range` = NULL key)
    unsigned long long* dspace;   // [dict_slots] accumulators addressed by dictionary entry (merged into `direct` after the batch)
    uint8_t* direct_valid;        // "holds a value" flags or nullptr
    uint8_t* dspace_valid;
};
struct FzLaunch {
    FzColumn col[FZ_MAX_COLS];
    FzAcc acc[FZ_MAX_ACCS];
    int32_t ncols, npred, key_col, nacc;
    int64_t n_rows;
    int32_t n_tiles;
    int32_t staged;                       // 1: tiles that qualify are done by the TMA-staged kernel, the tile kernel skips them
    long long kmin;
    int64_t range;
    uint8_t* seen_direct;
    uint8_t* seen_dspace;
    int32_t* oor;                         // a key outside [kmin, kmin + range): the column statistics were wrong
    unsigned long long* selected_rows;    // [0] rows that passed the predicates (FilterExec's output_rows), [1] tiles done by the staged kernel
    int32_t* left;                        // staged mode: [0] number of tiles left to the tile kernel, [1] next tile to hand out, then the tiles left
    // SUM(x), COUNT(x) of a narrow x (accumulators 0 and 1): rows whose key is a dictionary entry add ((1 << pack_shift) | (x - pack_bias))
    // to the entry's SUM word with ONE atomic -- the atomic unit, not the issue slots, bounds the kernel (1.29 cycles per lane
    // and SM); fz_merge splits the word.  pack_shift = 0: off.  x outside [pack_bias, pack_bias + 2^pack_bits) raises `oor`.
    int32_t pack_shift, pack_bits;
    long long pack_bias;
};
struct FzMerge {                  // dictionary space -> direct table, one launch per batch
    const PqDict* dicts;
    const int32_t* dslot_base;    // [n_dicts + 1]
    int32_t n_dicts, nacc;
    FzAcc acc[FZ_MAX_ACCS];
    long long kmin;
    int64_t range;
    uint8_t* seen_direct;
    const uint8_t* seen_dspace;
    int32_t* oor;
    int32_t pack_shift, pack_bits;    // as in FzLaunch
    long long pack_bias;
};
void fz_scout(Ctx& ctx, const std::vector<FzScoutCol>& cols);
void fz_dict_pass(Ctx& ctx, const PqDict* dicts, const int32_t* pass_off, int n_dicts, int total_words, int64_t lo, int64_t hi, uint32_t* pass_bits);
void fz_init_dspace(Ctx& ctx, const FzLaunch& L, int64_t dict_slots);
void fz_run(Ctx& ctx, const FzLaunch& L);
void fz_merge(Ctx& ctx, const FzMerge& M, int64_t dict_slots);

}  // namespace auron
