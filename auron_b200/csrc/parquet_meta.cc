// parquet_meta.cc -- Thrift compact protocol reader for the Parquet footer and page headers, and a
// Snappy block decompressor (host side of ParquetScanExec).
#include "parquet_meta.h"

#include <algorithm>
#include <cstring>

namespace auron {
namespace pq {

namespace {
struct TReader {
    const uint8_t* p;
    const uint8_t* end;
    const uint8_t* begin;
    TReader(const uint8_t* b, size_t n) : p(b), end(b + n), begin(b) {}
    uint8_t byte() {
        AURON_CHECK(p < end, "parquet: truncated thrift data");
        return *p++;
    }
    uint64_t varint() {
        uint64_t v = 0;
        int shift = 0;
        for (;;) {
            uint8_t b = byte();
            v |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) return v;
            shift += 7;
            AURON_CHECK(shift < 70, "parquet: malformed varint");
        }
    }
    int64_t zigzag() {
        uint64_t v = varint();
        return (int64_t)(v >> 1) ^ -(int64_t)(v & 1);
    }
    std::string binary() {
        uint64_t n = varint();
        AURON_CHECK((uint64_t)(end - p) >= n, "parquet: truncated binary");
        std::string s((const char*)p, (size_t)n);
        p += n;
        return s;
    }
    // field header; returns false on STOP
    bool field(int16_t* id, int* type, int16_t* last_id) {
        uint8_t h = byte();
        if (h == 0) return false;
        *type = h & 0x0f;
        int delta = h >> 4;
        if (delta == 0) *id = (int16_t)zigzag();
        else *id = (int16_t)(*last_id + delta);
        *last_id = *id;
        return true;
    }
    void list_header(int* elem_type, uint32_t* size) {
        uint8_t h = byte();
        *elem_type = h & 0x0f;
        *size = h >> 4;
        if (*size == 15) *size = (uint32_t)varint();
    }
    int depth = 0;   // nesting of skipped containers / structs (a footer of 0x1C bytes would otherwise recurse once per byte)
    struct DepthGuard {
        int& d;
        explicit DepthGuard(int& x) : d(x) { AURON_CHECK(++d <= 64, "parquet: thrift structure nested too deeply"); }
        ~DepthGuard() { --d; }
    };
    void skip(int type) {
        DepthGuard g(depth);
        switch (type) {
            case 1: case 2: break;   // bool in field header
            case 3: byte(); break;
            case 4: case 5: case 6: varint(); break;
            case 7: AURON_CHECK(end - p >= 8, "parquet: truncated double"); p += 8; break;
            case 8: binary(); break;
            case 9: case 10: {
                int et;
                uint32_t n;
                list_header(&et, &n);
                AURON_CHECK((size_t)(end - p) >= n, "parquet: truncated thrift list");
                for (uint32_t i = 0; i < n; i++) {
                    if (et == 1 || et == 2) byte();
                    else skip(et);
                }
                break;
            }
            case 11: {
                uint32_t n = (uint32_t)varint();
                if (n) {
                    uint8_t kv = byte();
                    AURON_CHECK((size_t)(end - p) >= n, "parquet: truncated thrift map");   // every entry takes at least one byte
                    for (uint32_t i = 0; i < n; i++) {
                        for (int et : {kv >> 4, kv & 0x0f}) {
                            if (et == 1 || et == 2) byte();   // bools inside containers are one byte each
                            else skip(et);
                        }
                    }
                }
                break;
            }
            case 12: {
                int16_t id, last = 0;
                int t;
                while (field(&id, &t, &last)) skip(t);
                break;
            }
            default: fail("parquet: unknown thrift type " + std::to_string(type));
        }
    }
};

// union LogicalType (parquet.thrift): 1 STRING, 5 DECIMAL{1 scale, 2 precision}, 6 DATE, 8 TIMESTAMP{1 isAdjustedToUTC, 2 unit},
// 10 INTEGER{1 bitWidth (i8), 2 isSigned}; TimeUnit: 1 MILLIS, 2 MICROS, 3 NANOS.  Every other member is LK_OTHER.
void read_logical_type(TReader& r, SchemaElement& e) {
    int16_t id, last = 0;
    int t;
    e.has_logical_type = true;
    e.logical = LK_OTHER;
    while (r.field(&id, &t, &last)) {
        if (t != 12) {
            r.skip(t);
            continue;
        }
        int16_t i2, l2 = 0;
        int t2;
        switch (id) {
            case 1: e.logical = LK_STRING; r.skip(t); break;
            case 2: e.map_annot = true; r.skip(t); break;
            case 3: e.list_annot = true; r.skip(t); break;
            case 6: e.logical = LK_DATE; r.skip(t); break;
            case 5:
                e.logical = LK_DECIMAL;
                while (r.field(&i2, &t2, &l2)) {
                    if (i2 == 1 && t2 == 5) e.scale = (int32_t)r.zigzag();
                    else if (i2 == 2 && t2 == 5) e.precision = (int32_t)r.zigzag();
                    else r.skip(t2);
                }
                break;
            case 8:
                e.logical = LK_TIMESTAMP;
                while (r.field(&i2, &t2, &l2)) {
                    if (i2 == 1 && (t2 == 1 || t2 == 2)) e.ts_utc = t2 == 1;   // a bool's value is its field type
                    else if (i2 == 2 && t2 == 12) {
                        int16_t i3, l3 = 0;
                        int t3;
                        while (r.field(&i3, &t3, &l3)) {
                            if (i3 >= 1 && i3 <= 3) e.ts_unit = i3;
                            r.skip(t3);
                        }
                    } else r.skip(t2);
                }
                if (e.ts_unit < 0) e.logical = LK_OTHER;
                break;
            case 10:
                e.logical = LK_INTEGER;
                while (r.field(&i2, &t2, &l2)) {
                    if (i2 == 1 && t2 == 3) e.int_bits = (int8_t)r.byte();
                    else if (i2 == 2 && (t2 == 1 || t2 == 2)) e.int_signed = t2 == 1;
                    else r.skip(t2);
                }
                if (e.int_bits != 8 && e.int_bits != 16 && e.int_bits != 32 && e.int_bits != 64) e.logical = LK_OTHER;
                break;
            default: r.skip(t);
        }
    }
}
// ConvertedType (parquet.thrift) -> annotation, for files without a LogicalType
void logical_from_converted(SchemaElement& e) {
    const int c = e.converted_type;
    if (c < 0) return;
    if (c == 0) e.logical = LK_STRING;
    else if (c == 5) e.logical = LK_DECIMAL;
    else if (c == 6) e.logical = LK_DATE;
    else if (c == 9 || c == 10) {   // TIMESTAMP_MILLIS / TIMESTAMP_MICROS: adjusted to UTC (LogicalTypes.md, "Backward compatibility")
        e.logical = LK_TIMESTAMP;
        e.ts_unit = c == 9 ? 1 : 2;
        e.ts_utc = true;
    } else if (c >= 11 && c <= 18) {   // UINT_8 .. UINT_64, INT_8 .. INT_64
        e.logical = LK_INTEGER;
        e.int_signed = c >= 15;
        e.int_bits = 8 << ((c - 11) % 4);
    } else if (c >= 1 && c <= 4) {
        e.logical = c == 4 ? LK_STRING : LK_OTHER;   // ENUM is a string; MAP / LIST belong to groups
    } else e.logical = LK_OTHER;
}

SchemaElement read_schema_element(TReader& r) {
    SchemaElement e;
    int16_t id, last = 0;
    int t;
    while (r.field(&id, &t, &last)) {
        switch (id) {
            case 1: e.type = (int32_t)r.zigzag(); break;
            case 2: e.type_length = (int32_t)r.zigzag(); break;
            case 3: e.repetition = (int32_t)r.zigzag(); break;
            case 4: e.name = r.binary(); break;
            case 5: e.num_children = (int32_t)r.zigzag(); break;
            case 6: e.converted_type = (int32_t)r.zigzag(); break;
            case 7: e.scale = (int32_t)r.zigzag(); break;
            case 8: e.precision = (int32_t)r.zigzag(); break;
            case 10:
                if (t == 12) read_logical_type(r, e);
                else r.skip(t);
                break;
            default: r.skip(t);
        }
    }
    if (!e.has_logical_type) logical_from_converted(e);
    if (e.converted_type == 3) e.list_annot = true;   // LIST
    if (e.converted_type == 1 || e.converted_type == 2) e.map_annot = true;   // MAP, MAP_KEY_VALUE
    return e;
}
Statistics read_statistics(TReader& r) {
    Statistics s;
    int16_t id, last = 0;
    int t;
    std::string old_min, old_max;
    bool has_old_min = false, has_old_max = false;
    while (r.field(&id, &t, &last)) {
        switch (id) {
            case 1: old_max = r.binary(); has_old_max = true; break;
            case 2: old_min = r.binary(); has_old_min = true; break;
            case 3: s.null_count = r.zigzag(); s.has_null_count = true; break;
            case 5: s.max_value = r.binary(); s.has_max = true; break;
            case 6: s.min_value = r.binary(); s.has_min = true; break;
            default: r.skip(t);
        }
    }
    if (!s.has_max && has_old_max) { s.max_value = old_max; s.has_max = s.legacy_max = true; }
    if (!s.has_min && has_old_min) { s.min_value = old_min; s.has_min = s.legacy_min = true; }
    return s;
}
ColumnMeta read_column_meta(TReader& r) {
    ColumnMeta m;
    int16_t id, last = 0;
    int t;
    while (r.field(&id, &t, &last)) {
        switch (id) {
            case 1: m.type = (int32_t)r.zigzag(); break;
            case 3: {
                int et;
                uint32_t n;
                r.list_header(&et, &n);
                for (uint32_t i = 0; i < n; i++) m.path.push_back(r.binary());
                break;
            }
            case 4: m.codec = (int32_t)r.zigzag(); break;
            case 5: m.num_values = r.zigzag(); break;
            case 6: m.total_uncompressed = r.zigzag(); break;
            case 7: m.total_compressed = r.zigzag(); break;
            case 9: m.data_page_offset = r.zigzag(); break;
            case 11: m.dictionary_page_offset = r.zigzag(); break;
            case 12: m.stats = read_statistics(r); break;
            default: r.skip(t);
        }
    }
    return m;
}
ColumnMeta read_column_chunk(TReader& r) {
    ColumnMeta m;
    int16_t id, last = 0;
    int t;
    while (r.field(&id, &t, &last)) {
        if (id == 3 && t == 12) m = read_column_meta(r);
        else r.skip(t);
    }
    return m;
}
RowGroup read_row_group(TReader& r) {
    RowGroup g;
    int16_t id, last = 0;
    int t;
    while (r.field(&id, &t, &last)) {
        switch (id) {
            case 1: {
                int et;
                uint32_t n;
                r.list_header(&et, &n);
                for (uint32_t i = 0; i < n; i++) g.columns.push_back(read_column_chunk(r));
                break;
            }
            case 2: g.total_byte_size = r.zigzag(); break;
            case 3: g.num_rows = r.zigzag(); break;
            case 5: g.file_offset = r.zigzag(); break;
            default: r.skip(t);
        }
    }
    return g;
}
}  // namespace

FileMeta parse_file_meta(const uint8_t* buf, size_t len) {
    TReader r(buf, len);
    FileMeta m;
    int16_t id, last = 0;
    int t;
    while (r.field(&id, &t, &last)) {
        switch (id) {
            case 1: m.version = (int32_t)r.zigzag(); break;
            case 2: {
                int et;
                uint32_t n;
                r.list_header(&et, &n);
                for (uint32_t i = 0; i < n; i++) m.schema.push_back(read_schema_element(r));
                break;
            }
            case 3: m.num_rows = r.zigzag(); break;
            case 4: {
                int et;
                uint32_t n;
                r.list_header(&et, &n);
                for (uint32_t i = 0; i < n; i++) m.row_groups.push_back(read_row_group(r));
                break;
            }
            case 6: m.created_by = r.binary(); break;
            default: r.skip(t);
        }
    }
    // The legacy min / max fields were written in signed byte order whatever the column's type: a reader must ignore them unless
    // the column's sort order is signed (parquet.thrift, Statistics).  Column chunk c belongs to the c-th leaf of the schema.
    std::vector<const SchemaElement*> leaves;
    for (size_t i = 1; i < m.schema.size(); i++)
        if (m.schema[i].num_children == 0) leaves.push_back(&m.schema[i]);
    for (auto& rg : m.row_groups)
        for (size_t c = 0; c < rg.columns.size(); c++) {
            Statistics& s = rg.columns[c].stats;
            if (c < leaves.size() && leaves[c]->signed_order()) continue;
            if (s.legacy_min) s.has_min = s.legacy_min = false, s.min_value.clear();
            if (s.legacy_max) s.has_max = s.legacy_max = false, s.max_value.clear();
        }
    return m;
}

const char* shape_name(int shape) {
    switch (shape) {
        case SHAPE_FLAT: return "primitive";
        case SHAPE_LIST: return "list";
        case SHAPE_STRUCT: return "struct";
        case SHAPE_MAP: return "map";
        case SHAPE_LIST_OF_LIST: return "list of lists";
        case SHAPE_LIST_OF_STRUCT: return "list of structs";
        case SHAPE_LIST_OF_MAP: return "list of maps";
        default: return "malformed list";
    }
}

namespace {
// pre-order walk of element i's subtree; returns the index behind it.  def / rep: levels of the parent.
size_t walk_node(const std::vector<SchemaElement>& s, size_t i, int field, const std::string& parent, int def, int rep, int depth, SchemaTree& t,
                 std::vector<std::vector<size_t>>& kids) {
    AURON_CHECK(i < s.size(), "parquet: the schema ends inside a group");
    AURON_CHECK(depth <= 64, "parquet: schema nested too deeply");
    const SchemaElement& e = s[i];
    AURON_CHECK(e.num_children >= 0 && (size_t)e.num_children < s.size(), "parquet: bad num_children in the schema");
    const std::string path = parent.empty() ? e.name : parent + "." + e.name;
    def += e.repetition != 0;   // OPTIONAL or REPEATED
    rep += e.repetition == 2;
    if (e.num_children == 0) {
        t.leaves.push_back(SchemaLeaf{(int32_t)t.leaves.size(), (int32_t)i, field, def, rep, path});
        return i + 1;
    }
    size_t j = i + 1;
    for (int c = 0; c < e.num_children; c++) {
        kids[i].push_back(j);
        j = walk_node(s, j, field, path, def, rep, depth + 1, t, kids);
    }
    return j;
}
}  // namespace

SchemaTree walk_schema(const FileMeta& m) {
    SchemaTree t;
    const auto& s = m.schema;
    AURON_CHECK(!s.empty(), "empty parquet schema");
    std::vector<std::vector<size_t>> kids(s.size());
    size_t j = 1;
    for (int c = 0; c < s[0].num_children; c++) {
        TopField f;
        f.element = (int32_t)j;
        AURON_CHECK(j < s.size(), "parquet: the schema ends inside the root");
        f.name = s[j].name;
        const int32_t first_leaf = (int32_t)t.leaves.size();
        j = walk_node(s, j, (int)t.fields.size(), "", 0, 0, 0, t, kids);
        const SchemaElement& e = s[(size_t)f.element];
        const int opt = e.repetition == 1 ? 1 : 0;
        auto list_of_leaf = [&] {
            f.shape = SHAPE_LIST;
            f.leaf = first_leaf;
            f.list_def = e.repetition == 2 ? 0 : opt;   // (a bare repeated field is a required list)
            f.elem_def = f.list_def + 1;
        };
        if (e.num_children == 0) {
            if (e.repetition == 2) list_of_leaf();   // a repeated primitive outside any LIST group: list<required element>
            else {
                f.shape = SHAPE_FLAT;
                f.leaf = first_leaf;
            }
        } else if (e.map_annot) {
            f.shape = SHAPE_MAP;
        } else if (e.repetition == 2) {
            f.shape = SHAPE_LIST_OF_STRUCT;   // a repeated group outside any LIST group: list<required struct>
        } else if (!e.list_annot) {
            f.shape = SHAPE_STRUCT;
        } else if (kids[(size_t)f.element].size() == 1 && s[kids[(size_t)f.element][0]].repetition == 2) {
            const size_t r = kids[(size_t)f.element][0];
            const SchemaElement& R = s[r];
            if (R.num_children == 0) list_of_leaf();   // 2-level: the repeated primitive is the element
            else if (R.num_children > 1 || R.name == "array" || R.name == e.name + "_tuple") f.shape = SHAPE_LIST_OF_STRUCT;   // the repeated group is the element
            else {   // 3-level: the repeated group's only field is the element, whatever the names
                const SchemaElement& E = s[kids[r][0]];
                if (E.num_children == 0) {
                    if (E.repetition == 2) f.shape = SHAPE_LIST_OF_LIST;
                    else list_of_leaf();
                } else if (E.list_annot || E.repetition == 2) f.shape = SHAPE_LIST_OF_LIST;
                else if (E.map_annot) f.shape = SHAPE_LIST_OF_MAP;
                else f.shape = SHAPE_LIST_OF_STRUCT;
            }
        } else {
            f.shape = SHAPE_OTHER;   // a LIST group must hold exactly one repeated field
        }
        t.fields.push_back(f);
    }
    AURON_CHECK(j == s.size(), "parquet: schema elements outside the root's tree");
    return t;
}

PageHeader parse_page_header(const uint8_t* buf, size_t len) {
    TReader r(buf, len);
    PageHeader h;
    int16_t id, last = 0;
    int t;
    while (r.field(&id, &t, &last)) {
        switch (id) {
            case 1: h.type = (int32_t)r.zigzag(); break;
            case 2: h.uncompressed_size = (int32_t)r.zigzag(); break;
            case 3: h.compressed_size = (int32_t)r.zigzag(); break;
            case 5: {   // DataPageHeader
                int16_t i2, l2 = 0;
                int t2;
                while (r.field(&i2, &t2, &l2)) {
                    switch (i2) {
                        case 1: h.num_values = (int32_t)r.zigzag(); break;
                        case 2: h.encoding = (int32_t)r.zigzag(); break;
                        case 3: h.def_encoding = (int32_t)r.zigzag(); break;
                        case 4: h.rep_encoding = (int32_t)r.zigzag(); break;
                        default: r.skip(t2);
                    }
                }
                break;
            }
            case 7: {   // DictionaryPageHeader
                int16_t i2, l2 = 0;
                int t2;
                while (r.field(&i2, &t2, &l2)) {
                    switch (i2) {
                        case 1: h.num_values = (int32_t)r.zigzag(); break;
                        case 2: h.encoding = (int32_t)r.zigzag(); break;
                        default: r.skip(t2);
                    }
                }
                break;
            }
            case 8: {   // DataPageHeaderV2
                int16_t i2, l2 = 0;
                int t2;
                while (r.field(&i2, &t2, &l2)) {
                    switch (i2) {
                        case 1: h.num_values = (int32_t)r.zigzag(); break;
                        case 2: h.num_nulls = (int32_t)r.zigzag(); break;
                        case 3: h.num_rows = (int32_t)r.zigzag(); break;
                        case 4: h.encoding = (int32_t)r.zigzag(); break;
                        case 5: h.def_bytes = (int32_t)r.zigzag(); break;
                        case 6: h.rep_bytes = (int32_t)r.zigzag(); break;
                        case 7: h.v2_compressed = (t2 == 1); break;
                        default: r.skip(t2);
                    }
                }
                break;
            }
            default: r.skip(t);
        }
    }
    h.header_len = (int32_t)(r.p - r.begin);
    return h;
}

// ------------------------------------------------------------------------------------------- snappy
void snappy_decompress(const uint8_t* in, size_t in_len, uint8_t* out, size_t out_len) {
    const uint8_t* p = in;
    const uint8_t* end = in + in_len;
    // preamble: uncompressed length varint
    uint64_t ulen = 0;
    int shift = 0;
    for (;;) {
        AURON_CHECK(p < end, "snappy: truncated preamble");
        uint8_t b = *p++;
        ulen |= (uint64_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) break;
        shift += 7;
    }
    AURON_CHECK(ulen == out_len, "snappy: uncompressed size mismatch");
    size_t o = 0;
    while (p < end) {
        uint8_t tag = *p++;
        uint32_t len, off;
        switch (tag & 3) {
            case 0: {   // literal
                len = (tag >> 2) + 1;
                if (len > 60) {
                    int nb = (int)len - 60;
                    AURON_CHECK(end - p >= nb, "snappy: truncated literal length");
                    len = 0;
                    for (int i = 0; i < nb; i++) len |= (uint32_t)p[i] << (8 * i);
                    len += 1;
                    p += nb;
                }
                AURON_CHECK((size_t)(end - p) >= len && o + len <= out_len, "snappy: literal overruns");
                memcpy(out + o, p, len);
                p += len;
                o += len;
                continue;
            }
            case 1:
                AURON_CHECK(p < end, "snappy: truncated copy1");
                len = ((tag >> 2) & 7) + 4;
                off = ((uint32_t)(tag >> 5) << 8) | *p++;
                break;
            case 2:
                AURON_CHECK(end - p >= 2, "snappy: truncated copy2");
                len = (tag >> 2) + 1;
                off = (uint32_t)p[0] | ((uint32_t)p[1] << 8);
                p += 2;
                break;
            default:
                AURON_CHECK(end - p >= 4, "snappy: truncated copy4");
                len = (tag >> 2) + 1;
                off = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
                p += 4;
        }
        AURON_CHECK(off != 0 && off <= o && o + len <= out_len, "snappy: bad copy");
        for (uint32_t i = 0; i < len; i++) out[o + i] = out[o + i - off];   // may overlap
        o += len;
    }
    AURON_CHECK(o == out_len, "snappy: short output");
}

// ------------------------------------------------------------------------------------------ host helpers of the scan
// Walk the elements of a raw Snappy block without decoding it (tags only).  True when the block is well formed up to
// `max_tokens` elements; then [0, *head_in) / [0, *head_out) are the compressed / uncompressed bytes up to and including the
// last back reference, and `pieces` are the literals after it (nothing refers back into them or reads them again).
bool snappy_split(const uint8_t* p, int64_t n, int64_t unc, int max_tokens, int64_t* head_in, int64_t* head_out, std::vector<LitPiece>* pieces) {
    int64_t i = 0, out = 0;
    uint64_t v = 0;
    for (int shift = 0;; shift += 7) {
        if (i >= n || shift > 28) return false;
        const uint8_t b = p[i++];
        v |= (uint64_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) break;
    }
    if ((int64_t)v != unc || unc <= 0) return false;
    pieces->clear();
    *head_in = i;
    *head_out = 0;
    for (int tok = 0; i < n; tok++) {
        if (tok >= max_tokens) return false;
        const uint8_t tag = p[i++];
        if ((tag & 3) == 0) {
            int64_t len = (tag >> 2) + 1;
            if (len > 60) {
                const int nb = (int)len - 60;
                if (i + nb > n) return false;
                uint32_t w = 0;
                for (int k = 0; k < nb; k++) w |= (uint32_t)p[i + k] << (8 * k);
                i += nb;
                len = (int64_t)w + 1;
            }
            if (len > n - i || len > unc - out) return false;
            pieces->push_back(LitPiece{i, len});
            i += len;
            out += len;
        } else {
            const int64_t len = (tag & 3) == 1 ? 4 + ((tag >> 2) & 7) : (tag >> 2) + 1;
            i += (tag & 3) == 1 ? 1 : (tag & 3) == 2 ? 2 : 4;
            if (i > n || len > unc - out) return false;
            out += len;
            pieces->clear();        // literals before a back reference belong to the head
            *head_in = i;
            *head_out = out;
        }
    }
    return out == unc;
}
static bool delta_varint(const uint8_t* p, size_t n, size_t& pos, uint64_t& v);
int64_t hybrid_count(const uint8_t* p, size_t n, int bw, int64_t num, uint32_t match) {
    AURON_CHECK(bw >= 0 && bw <= 8, "parquet: level bit width out of range");
    size_t pos = 0;
    int64_t seen = 0, hits = 0;
    while (seen < num) {
        uint64_t h = 0;
        AURON_CHECK(delta_varint(p, n, pos, h), "parquet: level stream ends early");
        if (h & 1) {   // bit-packed: (h >> 1) groups of 8 values
            const uint64_t groups = h >> 1;
            AURON_CHECK(groups <= (n - pos) && groups * (uint64_t)bw <= n - pos, "parquet: level stream ends early");
            const int64_t cnt = (int64_t)std::min<uint64_t>(groups * 8, (uint64_t)(num - seen));
            for (int64_t i = 0; i < cnt; i++) {
                uint32_t v = 0;
                for (int k = 0; k < bw; k++) {
                    const uint64_t b = (uint64_t)i * bw + k;
                    v |= (uint32_t)((p[pos + (b >> 3)] >> (b & 7)) & 1) << k;
                }
                hits += v == match;
            }
            seen += cnt;
            pos += (size_t)(groups * bw);
        } else {
            const uint64_t cnt = h >> 1;
            const int nb = (bw + 7) / 8;
            AURON_CHECK(cnt > 0 && pos + nb <= n, "parquet: malformed level run");
            uint32_t v = 0;
            for (int k = 0; k < nb; k++) v |= (uint32_t)p[pos + k] << (8 * k);
            pos += nb;
            const int64_t take = (int64_t)std::min<uint64_t>(cnt, (uint64_t)(num - seen));
            hits += v == match ? take : 0;
            seen += take;
        }
    }
    return hits;
}
// ---- DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY string pages are rewritten as PLAIN on the host (each value of the second
// depends on the bytes of the one before it; both are rare next to dictionary and PLAIN pages)
static bool delta_varint(const uint8_t* p, size_t n, size_t& pos, uint64_t& v) {
    v = 0;
    for (int shift = 0; shift < 70; shift += 7) {
        if (pos >= n) return false;
        const uint8_t b = p[pos++];
        v |= (uint64_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) return true;
    }
    return false;
}
// one DELTA_BINARY_PACKED stream at p[pos...] -> values; pos ends behind the stream
void delta_binary_decode(const uint8_t* p, size_t n, size_t& pos, std::vector<int64_t>& out, size_t max_values) {
    uint64_t bs = 0, nm = 0, total = 0, fv = 0;
    AURON_CHECK(delta_varint(p, n, pos, bs) && delta_varint(p, n, pos, nm) && delta_varint(p, n, pos, total) && delta_varint(p, n, pos, fv), "corrupt DELTA_BINARY_PACKED header");
    AURON_CHECK(nm > 0 && nm <= 512 && bs > 0 && bs <= (1u << 20) && bs % nm == 0 && (bs / nm) % 8 == 0 && total <= (uint64_t)max_values, "corrupt DELTA_BINARY_PACKED header");
    const size_t per_mini = (size_t)(bs / nm);
    out.clear();
    out.reserve((size_t)total);
    uint64_t last = (fv >> 1) ^ (0 - (fv & 1));
    if (total) out.push_back((int64_t)last);
    while (out.size() < total) {
        uint64_t md = 0;
        AURON_CHECK(delta_varint(p, n, pos, md) && pos + nm <= n, "corrupt DELTA_BINARY_PACKED block");
        const uint64_t min_delta = (md >> 1) ^ (0 - (md & 1));
        const uint8_t* widths = p + pos;
        pos += (size_t)nm;
        for (size_t m = 0; m < nm && out.size() < total; m++) {
            const unsigned bw = widths[m];
            const size_t bytes = per_mini * bw / 8;
            AURON_CHECK(bw <= 64 && pos + bytes <= n, "corrupt DELTA_BINARY_PACKED miniblock");
            for (size_t i = 0; i < per_mini && out.size() < total; i++) {
                uint64_t d = 0;
                const size_t bit = i * bw;
                for (unsigned k = 0; k < bw; k++) {
                    const size_t b = bit + k;
                    d |= (uint64_t)((p[pos + (b >> 3)] >> (b & 7)) & 1) << k;
                }
                last += min_delta + d;
                out.push_back((int64_t)last);
            }
            pos += bytes;
        }
    }
}
// value section of a DELTA_LENGTH_BYTE_ARRAY (`front_coded` false) or DELTA_BYTE_ARRAY page -> PLAIN ([u32 length][bytes] ...)
std::vector<uint8_t> delta_strings_to_plain(const uint8_t* p, size_t n, bool front_coded, int32_t* n_values, size_t max_values) {
    size_t pos = 0;
    std::vector<int64_t> prefix, lens;
    if (front_coded) delta_binary_decode(p, n, pos, prefix, max_values);
    delta_binary_decode(p, n, pos, lens, max_values);
    AURON_CHECK(!front_coded || prefix.size() == lens.size(), "corrupt DELTA_BYTE_ARRAY page");
    std::vector<uint8_t> out;
    size_t prev_at = 0, prev_len = 0;
    for (size_t i = 0; i < lens.size(); i++) {
        const int64_t pl = front_coded ? prefix[i] : 0, sl = lens[i];
        AURON_CHECK(pl >= 0 && sl >= 0 && (size_t)pl <= prev_len && pos <= n && (size_t)sl <= n - pos && pl + sl <= INT32_MAX && out.size() + 4 + (size_t)(pl + sl) <= (size_t)INT32_MAX,
                    "corrupt delta-encoded string page");
        const uint32_t len = (uint32_t)(pl + sl);
        const size_t at = out.size();
        out.resize(at + 4 + len);
        memcpy(out.data() + at, &len, 4);
        if (pl) memmove(out.data() + at + 4, out.data() + prev_at + 4, (size_t)pl);
        memcpy(out.data() + at + 4 + pl, p + pos, (size_t)sl);
        pos += (size_t)sl;
        prev_at = at;
        prev_len = len;
    }
    *n_values = (int32_t)lens.size();
    return out;
}

}  // namespace pq
}  // namespace auron
