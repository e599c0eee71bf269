// parquet_describe.cc -- what the engine's own Parquet metadata reader (parquet_meta.cc: Thrift compact protocol, page headers,
// Snappy block format) sees in a file, as JSON.  Host only: a diagnostic for integration work ("why does this file not scan?")
// and the way the footer / page-header parser is pinned on the CPU against an independent reader (tests/test_host_boundary.py).
#include <cstdio>
#include <cstring>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/auron_b200.h"
#include "parquet_meta.h"

namespace auron {
namespace {

std::string hex(const std::string& s) {
    static const char* d = "0123456789abcdef";
    std::string o;
    for (unsigned char c : s) {
        o.push_back(d[c >> 4]);
        o.push_back(d[c & 15]);
    }
    return o;
}
std::string quote(const std::string& s) {
    std::string o = "\"";
    for (char c : s) {
        if (c == '"' || c == '\\') o.push_back('\\');
        if ((unsigned char)c < 0x20) o += ' ';
        else o.push_back(c);
    }
    return o + "\"";
}
std::vector<uint8_t> read_range(FILE* f, int64_t off, int64_t len) {
    std::vector<uint8_t> b((size_t)len);
    AURON_CHECK(fseek(f, (long)off, SEEK_SET) == 0 && fread(b.data(), 1, (size_t)len, f) == (size_t)len, "short read");
    return b;
}

std::string describe(const char* path) {
    FILE* f = fopen(path, "rb");
    AURON_CHECK(f, std::string("cannot open ") + path);
    struct Closer {
        FILE* f;
        ~Closer() { fclose(f); }
    } closer{f};
    fseek(f, 0, SEEK_END);
    const int64_t size = ftell(f);
    AURON_CHECK(size >= 12, "not a parquet file");
    auto tail = read_range(f, size - 8, 8);
    AURON_CHECK(memcmp(tail.data() + 4, "PAR1", 4) == 0, "missing PAR1 magic");
    uint32_t flen;
    memcpy(&flen, tail.data(), 4);
    AURON_CHECK((int64_t)flen + 8 <= size, "corrupt footer length");
    auto footer = read_range(f, size - 8 - flen, flen);
    pq::FileMeta md = pq::parse_file_meta(footer.data(), footer.size());
    std::ostringstream o;
    o << "{\"version\":" << md.version << ",\"num_rows\":" << md.num_rows << ",\"created_by\":" << quote(md.created_by) << ",\"schema\":[";
    for (size_t i = 0; i < md.schema.size(); i++) {
        const auto& e = md.schema[i];
        o << (i ? "," : "") << "{\"name\":" << quote(e.name) << ",\"type\":" << e.type << ",\"type_length\":" << e.type_length << ",\"repetition\":" << e.repetition
          << ",\"num_children\":" << e.num_children << ",\"converted_type\":" << e.converted_type << ",\"scale\":" << e.scale << ",\"precision\":" << e.precision
          << ",\"has_logical_type\":" << (e.has_logical_type ? "true" : "false") << ",\"logical\":" << e.logical << ",\"ts_unit\":" << e.ts_unit
          << ",\"ts_utc\":" << (e.ts_utc ? "true" : "false") << ",\"int_bits\":" << e.int_bits << ",\"int_signed\":" << (e.int_signed ? "true" : "false") << "}";
    }
    // the schema as a tree: every leaf with its levels and the top-level field it belongs to (a schema that is not a tree is
    // described without it, as far as the flat walk goes)
    pq::SchemaTree tree;
    std::string tree_error;
    try {
        tree = pq::walk_schema(md);
    } catch (const std::exception& e) {
        tree_error = e.what();
        tree = pq::SchemaTree();
    }
    o << "],\"leaves\":[";
    for (size_t i = 0; i < tree.leaves.size(); i++) {
        const auto& l = tree.leaves[i];
        const auto& f = tree.fields[(size_t)l.field];
        o << (i ? "," : "") << "{\"path\":" << quote(l.path) << ",\"chunk\":" << l.chunk << ",\"element\":" << l.element << ",\"max_def\":" << l.max_def
          << ",\"max_rep\":" << l.max_rep << ",\"field\":" << quote(f.name) << ",\"shape\":" << quote(pq::shape_name(f.shape)) << ",\"read\":"
          << (f.leaf == (int32_t)i ? "true" : "false") << "}";
    }
    o << "],\"fields\":[";
    for (size_t i = 0; i < tree.fields.size(); i++) {
        const auto& f = tree.fields[i];
        o << (i ? "," : "") << "{\"name\":" << quote(f.name) << ",\"shape\":" << quote(pq::shape_name(f.shape)) << ",\"leaf\":" << f.leaf
          << ",\"list_def\":" << f.list_def << ",\"elem_def\":" << f.elem_def << "}";
    }
    o << "]";
    if (!tree_error.empty()) o << ",\"schema_error\":" << quote(tree_error);
    o << ",\"row_groups\":[";
    for (size_t g = 0; g < md.row_groups.size(); g++) {
        const auto& rg = md.row_groups[g];
        o << (g ? "," : "") << "{\"num_rows\":" << rg.num_rows << ",\"total_byte_size\":" << rg.total_byte_size << ",\"columns\":[";
        for (size_t c = 0; c < rg.columns.size(); c++) {
            const auto& cm = rg.columns[c];
            std::string path_in_schema;
            for (size_t k = 0; k < cm.path.size(); k++) path_in_schema += (k ? "." : "") + cm.path[k];
            o << (c ? "," : "") << "{\"path\":" << quote(path_in_schema) << ",\"type\":" << cm.type << ",\"codec\":" << cm.codec << ",\"num_values\":" << cm.num_values
              << ",\"total_uncompressed\":" << cm.total_uncompressed << ",\"total_compressed\":" << cm.total_compressed << ",\"data_page_offset\":" << cm.data_page_offset
              << ",\"dictionary_page_offset\":" << cm.dictionary_page_offset;
            if (cm.stats.has_min) o << ",\"min\":\"" << hex(cm.stats.min_value) << "\"";
            if (cm.stats.has_max) o << ",\"max\":\"" << hex(cm.stats.max_value) << "\"";
            if (cm.stats.has_null_count) o << ",\"null_count\":" << cm.stats.null_count;
            // walk the page chain of the chunk: headers must tile the chunk exactly; SNAPPY bodies are decompressed with the
            // engine's own block decoder as a check of sizes
            auto chunk = read_range(f, cm.start_offset(), cm.total_compressed);
            int64_t pos = 0, values = 0, pages = 0, dict_pages = 0, unc = 0, snappy_checked = 0;
            // the scan's host-side helpers, exercised here on the CPU: the tag walk that splits a Snappy body into a head and stored
            // literal pieces (checked against the decompressed body), and the decoders of the DELTA encodings (count + wrapping sum of
            // the integers, count + byte total + FNV-1a of the PLAIN transcription of the strings)
            int64_t split_pages = 0, split_head_out = 0, split_stored = 0, delta_pages = 0, delta_values = 0, delta_bytes = 0;
            uint64_t delta_sum = 0, delta_fnv = 1469598103934665603ull;
            // levels of the chunk's leaf (a schema that is not a tree: element c + 1, as for a flat schema)
            const int max_def = c < tree.leaves.size() ? tree.leaves[c].max_def : (c + 1 < md.schema.size() && md.schema[c + 1].repetition == 1) ? 1 : 0;
            const int max_rep = c < tree.leaves.size() ? tree.leaves[c].max_rep : 0;
            int64_t level_pages = 0, level_rows = 0, level_values = 0;
            std::string encodings;
            while (pos < cm.total_compressed) {
                pq::PageHeader h = pq::parse_page_header(chunk.data() + pos, (size_t)(cm.total_compressed - pos));
                AURON_CHECK(pos + h.header_len + h.compressed_size <= cm.total_compressed, "page overruns its column chunk");
                const uint8_t* body = chunk.data() + pos + h.header_len;
                if (h.type == pq::PAGE_DICTIONARY) dict_pages++;
                else if (h.type == pq::PAGE_DATA || h.type == pq::PAGE_DATA_V2) {
                    pages++;
                    values += h.num_values;
                    const std::string e = std::to_string(h.encoding);
                    if (("," + encodings + ",").find("," + e + ",") == std::string::npos) encodings += (encodings.empty() ? "" : ",") + e;
                }
                unc += h.uncompressed_size + h.header_len;
                const int lvl = h.type == pq::PAGE_DATA_V2 ? h.def_bytes + h.rep_bytes : 0;
                std::vector<uint8_t> out;   // uncompressed body behind the v2 level bytes (SNAPPY and UNCOMPRESSED chunks)
                bool have_body = false;
                if (cm.codec == pq::CODEC_SNAPPY && !(h.type == pq::PAGE_DATA_V2 && !h.v2_compressed) && h.uncompressed_size > lvl) {
                    out.resize((size_t)(h.uncompressed_size - lvl) + 8);
                    pq::snappy_decompress(body + lvl, (size_t)(h.compressed_size - lvl), out.data(), (size_t)(h.uncompressed_size - lvl));
                    snappy_checked++;
                    have_body = true;
                    std::vector<pq::LitPiece> pieces;
                    int64_t head_in = 0, head_out = 0;
                    const int64_t body_out = h.uncompressed_size - lvl;
                    if (pq::snappy_split(body + lvl, h.compressed_size - lvl, body_out, 4096, &head_in, &head_out, &pieces) && !pieces.empty()) {
                        int64_t at = head_out;
                        for (auto& pc : pieces) {   // the literals behind the last back reference must be the tail of the body, byte for byte
                            AURON_CHECK(at + pc.len <= body_out && memcmp(out.data() + at, body + lvl + pc.src_off, (size_t)pc.len) == 0, "snappy_split: a literal piece does not match the decompressed body");
                            at += pc.len;
                        }
                        AURON_CHECK(at == body_out, "snappy_split: the pieces do not end at the end of the body");
                        split_pages++;
                        split_head_out += head_out;
                        split_stored += body_out - head_out;
                    }
                } else if ((cm.codec == pq::CODEC_UNCOMPRESSED || (h.type == pq::PAGE_DATA_V2 && !h.v2_compressed)) && h.uncompressed_size > lvl && h.compressed_size > lvl) {
                    out.assign(body + lvl, body + h.compressed_size);
                    out.resize(out.size() + 8);
                    have_body = true;
                }
                const size_t blen = have_body ? out.size() - 8 : 0;   // bytes of `out` that belong to the page (sizes in a damaged header are not trusted)
                // leaves under a repeated field: rows (rep == 0) and non-null values (def == max_def) of the page, counted from its levels with
                // the walk the scan uses for v1 list pages
                if (max_rep > 0 && (h.type == pq::PAGE_DATA || h.type == pq::PAGE_DATA_V2)) {
                    const uint8_t *rp = nullptr, *dp = nullptr;
                    size_t rl = 0, dl = 0;
                    if (h.type == pq::PAGE_DATA_V2) {
                        AURON_CHECK(h.rep_bytes >= 0 && h.def_bytes >= 0 && (int64_t)h.rep_bytes + h.def_bytes <= h.compressed_size, "corrupt parquet page levels");
                        rp = body, rl = (size_t)h.rep_bytes, dp = body + h.rep_bytes, dl = (size_t)h.def_bytes;
                    } else if (have_body) {
                        uint32_t a = 0, b = 0;
                        AURON_CHECK(blen >= 4, "corrupt parquet page");
                        memcpy(&a, out.data(), 4);
                        AURON_CHECK((size_t)a + 8 <= blen, "corrupt parquet page levels");
                        memcpy(&b, out.data() + 4 + a, 4);
                        AURON_CHECK((size_t)a + 8 + b <= blen, "corrupt parquet page levels");
                        rp = out.data() + 4, rl = a, dp = out.data() + 8 + a, dl = b;
                    }
                    if (rp) {
                        auto bw = [](int m) { int b = 0; while ((1 << b) <= m) b++; return b; };
                        level_rows += pq::hybrid_count(rp, rl, bw(max_rep), h.num_values, 0);
                        level_values += pq::hybrid_count(dp, dl, bw(max_def), h.num_values, (uint32_t)max_def);
                        level_pages++;
                    }
                }
                const bool delta = h.encoding == pq::ENC_DELTA_BINARY_PACKED || h.encoding == pq::ENC_DELTA_LENGTH_BYTE_ARRAY || h.encoding == pq::ENC_DELTA_BYTE_ARRAY;
                if (have_body && delta && (h.type == pq::PAGE_DATA || h.type == pq::PAGE_DATA_V2)) {
                    size_t vo = 0;   // value section inside `out`
                    if (h.type == pq::PAGE_DATA)   // [u32 length][repetition levels] if max_rep > 0, [u32 length][definition levels] if max_def > 0
                        for (int sec = (max_rep > 0 ? 0 : 1); sec < (max_def > 0 ? 2 : 1); sec++) {
                            AURON_CHECK(vo + 4 <= blen, "corrupt parquet page");
                            uint32_t dl = 0;
                            memcpy(&dl, out.data() + vo, 4);
                            vo += 4 + (size_t)dl;
                        }
                    AURON_CHECK(vo <= blen && h.num_values >= 0, "corrupt parquet page levels");
                    const size_t vlen = blen - vo;
                    if (h.encoding == pq::ENC_DELTA_BINARY_PACKED) {
                        std::vector<int64_t> vals;
                        size_t dp = 0;
                        pq::delta_binary_decode(out.data() + vo, vlen, dp, vals, (size_t)h.num_values);
                        delta_values += (int64_t)vals.size();
                        for (int64_t v : vals) delta_sum += (uint64_t)(cm.type == pq::PT_INT32 ? (int64_t)(int32_t)v : v);
                    } else {
                        int32_t nv = 0;
                        const std::vector<uint8_t> plain = pq::delta_strings_to_plain(out.data() + vo, vlen, h.encoding == pq::ENC_DELTA_BYTE_ARRAY, &nv, (size_t)h.num_values);
                        delta_values += nv;
                        delta_bytes += (int64_t)plain.size() - 4 * (int64_t)nv;
                        size_t q = 0;
                        for (int32_t k = 0; k < nv; k++) {   // FNV-1a over the value bytes, a 0xFF between values
                            uint32_t len;
                            memcpy(&len, plain.data() + q, 4);
                            q += 4;
                            for (uint32_t b = 0; b < len; b++) delta_fnv = (delta_fnv ^ plain[q + b]) * 1099511628211ull;
                            delta_fnv = (delta_fnv ^ 0xFFu) * 1099511628211ull;
                            q += len;
                        }
                    }
                    delta_pages++;
                }
                pos += h.header_len + h.compressed_size;
            }
            AURON_CHECK(pos == cm.total_compressed, "page headers do not tile the column chunk");
            o << ",\"data_pages\":" << pages << ",\"dictionary_pages\":" << dict_pages << ",\"page_values\":" << values << ",\"pages_uncompressed\":" << unc
              << ",\"snappy_pages_decompressed\":" << snappy_checked << ",\"snappy_split_pages\":" << split_pages << ",\"snappy_split_head_bytes\":" << split_head_out
              << ",\"snappy_split_stored_bytes\":" << split_stored << ",\"delta_pages\":" << delta_pages << ",\"delta_values\":" << delta_values << ",\"delta_sum\":\""
              << delta_sum << "\",\"delta_string_bytes\":" << delta_bytes << ",\"delta_fnv\":\"" << delta_fnv << "\",\"page_encodings\":[" << encodings << "]";
            if (max_rep > 0) o << ",\"level_pages\":" << level_pages << ",\"level_rows\":" << level_rows << ",\"level_values\":" << level_values;
            o << "}";
        }
        o << "]}";
    }
    o << "]}";
    return o.str();
}

thread_local std::string g_describe_error;

}  // namespace
}  // namespace auron

extern "C" __attribute__((visibility("default"))) int64_t auron_b200_parquet_describe(const char* path, char* out, int64_t cap) {
    try {
        const std::string s = auron::describe(path);
        if (out && cap > 0) {
            const size_t n = std::min<size_t>(s.size(), (size_t)cap - 1);
            memcpy(out, s.data(), n);
            out[n] = 0;
        }
        return (int64_t)s.size();
    } catch (const std::exception& e) {
        if (out && cap > 0) {
            snprintf(out, (size_t)cap, "%s", e.what());
        }
        return -1;
    } catch (...) {
        return -1;
    }
}
