// parquet_meta.h -- Parquet footer / page-header structures and their Thrift compact-protocol parser.
// The reference delegates all of this to the third-party `parquet` crate 55.2 (arrow-rs fork rev 5de02520c,
// Cargo.toml:211-224; call site datafusion-ext-plans/src/parquet_exec.rs:175-197); the structures below
// follow the published parquet-format Thrift definition (parquet.thrift), restated by field id.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "common.h"

namespace auron {
namespace pq {

enum PhysType { PT_BOOLEAN = 0, PT_INT32 = 1, PT_INT64 = 2, PT_INT96 = 3, PT_FLOAT = 4, PT_DOUBLE = 5, PT_BYTE_ARRAY = 6, PT_FLBA = 7 };
enum Encoding { ENC_PLAIN = 0, ENC_PLAIN_DICTIONARY = 2, ENC_RLE = 3, ENC_BIT_PACKED = 4, ENC_DELTA_BINARY_PACKED = 5, ENC_DELTA_LENGTH_BYTE_ARRAY = 6, ENC_DELTA_BYTE_ARRAY = 7, ENC_RLE_DICTIONARY = 8 };
enum Codec { CODEC_UNCOMPRESSED = 0, CODEC_SNAPPY = 1, CODEC_GZIP = 2, CODEC_LZ4 = 5, CODEC_ZSTD = 6, CODEC_LZ4_RAW = 7 };
enum PageType { PAGE_DATA = 0, PAGE_INDEX = 1, PAGE_DICTIONARY = 2, PAGE_DATA_V2 = 3 };

// The annotation of a column: SchemaElement.logicalType (field 10) when present, else the one its converted_type (field 6) implies
enum LogicalKind { LK_NONE = 0, LK_STRING = 1, LK_DECIMAL = 2, LK_DATE = 3, LK_TIMESTAMP = 4, LK_INTEGER = 5, LK_OTHER = 6 };
struct SchemaElement {
    int32_t type = -1, type_length = 0, repetition = 0, num_children = 0, converted_type = -1, scale = 0, precision = 0;
    std::string name;
    bool has_logical_type = false;   // field 10 was present
    int32_t logical = LK_NONE;
    int32_t ts_unit = -1;            // LK_TIMESTAMP: 1 ms, 2 us, 3 ns (the coding of DType::unit)
    bool ts_utc = false;             // LK_TIMESTAMP: isAdjustedToUTC
    int32_t int_bits = 0;            // LK_INTEGER: 8, 16, 32 or 64
    bool int_signed = true;          // LK_INTEGER
    bool list_annot = false, map_annot = false;   // groups: LIST / MAP (or MAP_KEY_VALUE), from logicalType or converted_type
    // min / max statistics are ordered as signed values (the only order the legacy min / max fields may be read in)
    bool signed_order() const {
        if (logical == LK_INTEGER) return int_signed;
        if (logical == LK_DECIMAL) return true;
        return logical != LK_STRING && logical != LK_OTHER && type != 3 && type != 6 && type != 7 && type >= 0;
    }
};
struct Statistics {
    bool has_min = false, has_max = false, has_null_count = false;
    bool legacy_min = false, legacy_max = false;   // taken from the deprecated min / max fields (1, 2)
    std::string min_value, max_value;
    int64_t null_count = 0;
};
struct ColumnMeta {
    int32_t type = 0, codec = 0;
    std::vector<std::string> path;
    int64_t num_values = 0, total_uncompressed = 0, total_compressed = 0;
    int64_t data_page_offset = 0, dictionary_page_offset = -1;
    Statistics stats;
    int64_t start_offset() const { return dictionary_page_offset > 0 && dictionary_page_offset < data_page_offset ? dictionary_page_offset : data_page_offset; }
};
struct RowGroup {
    std::vector<ColumnMeta> columns;
    int64_t num_rows = 0, total_byte_size = 0, file_offset = -1;
};
struct FileMeta {
    int32_t version = 0;
    int64_t num_rows = 0;
    std::vector<SchemaElement> schema;
    std::vector<RowGroup> row_groups;
    std::string created_by;
};
struct PageHeader {
    int32_t type = 0, uncompressed_size = 0, compressed_size = 0;
    // data page (v1 / v2)
    int32_t num_values = 0, encoding = 0, def_encoding = 3, rep_encoding = 3;
    int32_t num_nulls = 0, num_rows = 0, def_bytes = 0, rep_bytes = 0;
    bool v2_compressed = true;
    int32_t header_len = 0;   // bytes consumed by the header itself
};

// ---- the schema as a tree (parquet-format LogicalTypes.md, "Nested Types" and its backward-compatibility rules)
// What the scan makes of one top-level field.  Only FLAT and LIST (a one-level list of a primitive) are read.
enum FieldShape { SHAPE_FLAT = 0, SHAPE_LIST = 1, SHAPE_STRUCT = 2, SHAPE_MAP = 3, SHAPE_LIST_OF_LIST = 4, SHAPE_LIST_OF_STRUCT = 5, SHAPE_LIST_OF_MAP = 6,
                  SHAPE_OTHER = 7 };
const char* shape_name(int shape);
struct SchemaLeaf {
    int32_t chunk;        // column-chunk index in every row group (leaves are numbered in schema order)
    int32_t element;      // index into FileMeta::schema
    int32_t field;        // index into SchemaTree::fields of the top-level field it belongs to
    int32_t max_def, max_rep;
    std::string path;     // dotted path from the root (ColumnMetaData.path_in_schema)
};
struct TopField {
    int32_t element;      // index into FileMeta::schema
    std::string name;
    int32_t shape = SHAPE_OTHER;
    int32_t leaf = -1;    // SHAPE_FLAT: its leaf; SHAPE_LIST: the element's leaf (index into SchemaTree::leaves)
    // SHAPE_LIST: a level slot with def < list_def is a NULL list, one with def < elem_def an empty list, every other slot holds an
    // element, NULL unless def == the leaf's max_def
    int32_t list_def = 0, elem_def = 0;
};
struct SchemaTree {
    std::vector<SchemaLeaf> leaves;
    std::vector<TopField> fields;
};
// throws auron::Error when the element list is not a tree rooted at element 0
SchemaTree walk_schema(const FileMeta& m);

// throws auron::Error on malformed input
FileMeta parse_file_meta(const uint8_t* buf, size_t len);
PageHeader parse_page_header(const uint8_t* buf, size_t len);

// raw snappy block decompression (format description: snappy framing-less block format)
void snappy_decompress(const uint8_t* in, size_t in_len, uint8_t* out, size_t out_len);

// ---- host helpers of the scan (scan_parquet.cc), here so that auron_b200_parquet_describe can exercise them on the CPU
struct LitPiece {
    int64_t src_off, len;
};
// Walks the elements of a raw Snappy block by their tags only.  True when the block is well formed within `max_tokens` elements; then
// [0, *head_in) / [0, *head_out) are the compressed / uncompressed bytes up to and including the last back reference and `pieces` the
// literals behind it (offsets into p).
bool snappy_split(const uint8_t* p, int64_t n, int64_t unc, int max_tokens, int64_t* head_in, int64_t* head_out, std::vector<LitPiece>* pieces);
// How many of the first `num` values of an RLE / bit-packed hybrid stream of bit width `bw` at p[0, n) equal `match` (the rows of a
// list page: rep == 0; its non-null values: def == max_def).  Throws when the stream ends early.
int64_t hybrid_count(const uint8_t* p, size_t n, int bw, int64_t num, uint32_t match);
// one DELTA_BINARY_PACKED stream at p[pos...] -> values; pos ends behind the stream
// (a stream may not announce more than `max_values` values: the page header's count -- zero-width miniblocks cost no input bytes)
void delta_binary_decode(const uint8_t* p, size_t n, size_t& pos, std::vector<int64_t>& out, size_t max_values);
// value section of a DELTA_LENGTH_BYTE_ARRAY (`front_coded` false) or DELTA_BYTE_ARRAY page -> PLAIN ([u32 length][bytes] ...)
std::vector<uint8_t> delta_strings_to_plain(const uint8_t* p, size_t n, bool front_coded, int32_t* n_values, size_t max_values);
}  // namespace pq
}  // namespace auron
