// planner.cc -- protobuf TaskDefinition -> operator tree.  Mirror of PhysicalPlanner::create_plan
// (auron-planner/src/planner.rs:120-842), try_parse_physical_expr (:844-1053) and the ArrowType / Schema /
// ScalarValue conversions (auron-planner/src/lib.rs).  Field numbers are those of
// auron-planner/proto/auron.proto; the wire format is decoded by hand (pb.h).
#include "operators.h"
#include "pb.h"

namespace auron {

// ------------------------------------------------------------------------------------------ types
static Field decode_field(const uint8_t* b, size_t n);
DType decode_arrow_type(const uint8_t* b, size_t n) {
    PbReader r(b, n);
    uint32_t f, w;
    DType t(T_NULL);
    while (r.next(&f, &w)) {
        const uint8_t* sb = nullptr;
        size_t sn = 0;
        uint64_t v = 0;
        if (w == 2) r.bytes_view(&sb, &sn);
        else if (w == 0) v = r.varint();
        else r.skip(w);
        switch (f) {   // auron.proto:915-951
            case 1: t = DType(T_NULL); break;
            case 2: t = DType(T_BOOL); break;
            case 4: t = DType(T_INT8); break;
            case 6: t = DType(T_INT16); break;
            case 8: t = DType(T_INT32); break;
            case 10: t = DType(T_INT64); break;
            case 12: t = DType(T_FLOAT32); break;
            case 13: t = DType(T_FLOAT64); break;
            case 14: case 32: t = DType(T_UTF8); break;
            case 15: case 31: t = DType(T_BINARY); break;
            case 17: t = DType(T_DATE32); break;
            case 18: t = DType(T_DATE64); break;
            case 20: {   // Timestamp{time_unit=1, timezone=2}
                t = DType(T_TIMESTAMP);
                t.unit = 0;
                PbReader tr(sb, sn);
                uint32_t tf, tw;
                while (tr.next(&tf, &tw)) {
                    if (tf == 1 && tw == 0) t.unit = (int)tr.varint();
                    else if (tf == 2 && tw == 2) t.tz = tr.bytes();
                    else tr.skip(tw);
                }
                break;
            }
            case 24: {   // Decimal{whole=1 (precision), fractional=2 (scale)}
                int p = 0, s = 0;
                PbReader dr(sb, sn);
                uint32_t df, dw;
                while (dr.next(&df, &dw)) {
                    if (df == 1 && dw == 0) p = (int)dr.varint();
                    else if (df == 2 && dw == 0) s = (int)(int64_t)dr.varint();
                    else dr.skip(dw);
                }
                t = DType::decimal(p, s);
                break;
            }
            case 3: case 5: case 7: case 9: fail("unsigned integer columns are not supported on device");
            case 25: {   // List{field_type=1}: one level of a flat element type
                Field e;
                PbReader lr(sb, sn);
                uint32_t lf, lw;
                bool has = false;
                while (lr.next(&lf, &lw)) {
                    if (lf == 1 && lw == 2) {
                        const uint8_t* eb;
                        size_t en;
                        lr.bytes_view(&eb, &en);
                        e = decode_field(eb, en);
                        has = true;
                    } else lr.skip(lw);
                }
                AURON_CHECK(has, "ArrowType list without its element field");
                if (e.type.id == T_LIST) fail("unsupported ArrowType list of list (tag 25): nested types are out of scope");
                t = DType::list(e.type, e.nullable, e.name);
                break;
            }
            case 26: case 27: fail("unsupported ArrowType list (tag " + std::to_string(f) + "): nested types are out of scope");
            case 28: case 33: fail(std::string("unsupported ArrowType ") + (f == 28 ? "struct" : "map") + " (tag " + std::to_string(f) + "): nested types are out of scope");
            default: fail("unsupported ArrowType tag " + std::to_string(f) + " (nested / interval types are out of scope)");
        }
        (void)v;
    }
    return t;
}

static Field decode_field(const uint8_t* b, size_t n) {
    PbReader r(b, n);
    uint32_t f, w;
    Field out;
    out.nullable = false;
    while (r.next(&f, &w)) {
        if (f == 1 && w == 2) out.name = r.bytes();
        else if (f == 2 && w == 2) {
            const uint8_t* sb;
            size_t sn;
            r.bytes_view(&sb, &sn);
            out.type = decode_arrow_type(sb, sn);
        } else if (f == 3 && w == 0) out.nullable = r.varint() != 0;
        else r.skip(w);
    }
    return out;
}
Schema decode_schema(const uint8_t* b, size_t n) {
    PbReader r(b, n);
    uint32_t f, w;
    Schema s;
    while (r.next(&f, &w)) {
        if (f == 1 && w == 2) {
            const uint8_t* sb;
            size_t sn;
            r.bytes_view(&sb, &sn);
            s.fields.push_back(decode_field(sb, sn));
        } else r.skip(w);
    }
    return s;
}

// ------------------------------------------------------------------------------------------ literals
// Arrow IPC stream: schema message + one record batch with one row / one column (NativeConverters.scala:413-428)
static bool next_ipc_message(const uint8_t*& p, const uint8_t* end, const uint8_t** meta, uint32_t* meta_len, const uint8_t** body, int64_t* body_len) {
    if (end - p < 4) return false;
    uint32_t first;
    memcpy(&first, p, 4);
    if (first == 0xFFFFFFFFu) {
        p += 4;
        if (end - p < 4) return false;
        memcpy(&first, p, 4);
    }
    p += 4;
    if (first == 0) return false;   // end-of-stream marker
    AURON_CHECK((size_t)(end - p) >= first, "Arrow IPC: truncated message");
    *meta = p;
    *meta_len = first;
    p += first;
    FbTable msg = FbTable::root(*meta, first);
    *body_len = msg.scalar<int64_t>(3, 0);
    *body = p;
    AURON_CHECK(*body_len >= 0 && end - p >= *body_len, "Arrow IPC: truncated body");
    p += *body_len;
    return true;
}

// org.apache.arrow.flatbuf.Field -> DType (flat types only)
static DType fb_field_type(const FbTable& field) {
    uint8_t tt = field.scalar<uint8_t>(2, 0);
    FbTable ty = field.table(3);
    DType t;
    switch (tt) {   // org.apache.arrow.flatbuf.Type
        case 1: t = DType(T_NULL); break;
        case 2: {
            int bw = ty.ok() ? ty.scalar<int32_t>(0, 0) : 0;
            bool sg = ty.ok() ? ty.scalar<uint8_t>(1, 0) != 0 : true;
            AURON_CHECK(sg, "unsigned literal");
            t = DType(bw == 8 ? T_INT8 : bw == 16 ? T_INT16 : bw == 32 ? T_INT32 : T_INT64);
            break;
        }
        case 3: {
            int prec = ty.ok() ? ty.scalar<int16_t>(0, 0) : 0;
            AURON_CHECK(prec == 1 || prec == 2, "half-float literal");
            t = DType(prec == 1 ? T_FLOAT32 : T_FLOAT64);
            break;
        }
        case 4: t = DType(T_BINARY); break;
        case 5: t = DType(T_UTF8); break;
        case 6: t = DType(T_BOOL); break;
        case 7: t = DType::decimal(ty.ok() ? ty.scalar<int32_t>(0, 0) : 0, ty.ok() ? ty.scalar<int32_t>(1, 0) : 0); break;
        case 8: t = DType((ty.ok() ? ty.scalar<int16_t>(0, 1) : 1) == 0 ? T_DATE32 : T_DATE64); break;
        case 10: {
            t = DType(T_TIMESTAMP);
            t.unit = ty.ok() ? ty.scalar<int16_t>(0, 0) : 0;
            if (ty.ok()) t.tz = ty.str(1);
            break;
        }
        default: fail("ScalarValue: unsupported literal type tag " + std::to_string(tt));
    }
    return t;
}

// ScalarValue holding a List<T> with ONE row (range partition bounds, planner.rs:1174-1203): returns the child array
HostArray decode_list_scalar_ipc(const uint8_t* bytes, size_t n) {
    const uint8_t* p = bytes;
    const uint8_t* end = bytes + n;
    const uint8_t *meta, *body;
    uint32_t meta_len;
    int64_t body_len;
    HostArray out;
    AURON_CHECK(next_ipc_message(p, end, &meta, &meta_len, &body, &body_len), "list ScalarValue: missing schema message");
    FbTable msg = FbTable::root(meta, meta_len);
    AURON_CHECK(msg.scalar<uint8_t>(1, 0) == 1, "list ScalarValue: first IPC message is not a Schema");
    FbTable schema = msg.table(2);
    AURON_CHECK(schema.ok(), "list ScalarValue: Schema message without a header");
    uint32_t nfields;
    const uint8_t* fields = schema.vec(1, &nfields);
    AURON_CHECK(nfields == 1, "list ScalarValue: expected exactly one field");
    FbTable field = schema.vec_table(fields, 0);
    uint8_t tt = field.scalar<uint8_t>(2, 0);
    AURON_CHECK(tt == 12 || tt == 21, "range partition bounds must be List scalars");   // List / LargeList
    AURON_CHECK(tt == 12, "LargeList bounds are not supported");
    uint32_t nchildren;
    const uint8_t* children = field.vec(5, &nchildren);
    AURON_CHECK(children && nchildren == 1, "list ScalarValue: malformed child field");
    const FbTable elem = field.vec_table(children, 0);
    out.type = fb_field_type(elem);
    out.elem_name = elem.str(0);
    out.elem_nullable = elem.scalar<uint8_t>(1, 0) != 0;
    AURON_CHECK(next_ipc_message(p, end, &meta, &meta_len, &body, &body_len), "list ScalarValue: missing record batch");
    msg = FbTable::root(meta, meta_len);
    AURON_CHECK(msg.scalar<uint8_t>(1, 0) == 3, "list ScalarValue: second IPC message is not a RecordBatch");
    FbTable rb = msg.table(2);
    AURON_CHECK(rb.ok(), "list ScalarValue: RecordBatch message without a header");
    uint32_t nnodes, nbufs;
    const uint8_t* nodes = rb.vec(1, &nnodes, 16);   // FieldNode{length, null_count}
    const uint8_t* bufs = rb.vec(2, &nbufs, 16);     // Buffer{offset, length}
    AURON_CHECK(rb.field_off(3) == 0, "list ScalarValue: compressed IPC bodies are not supported");
    AURON_CHECK(nnodes == 2 && rb.scalar<int64_t>(0, 0) == 1, "list ScalarValue: expected one list row");
    if (FbTable::rd<int64_t>(nodes + 8) > 0) {   // the list row is NULL: no elements
        out.list_is_null = true;
        return out;
    }
    auto buf = [&](uint32_t i, int64_t* len) -> const uint8_t* {
        AURON_CHECK(i < nbufs, "list ScalarValue: missing buffer");
        int64_t off = FbTable::rd<int64_t>(bufs + 16 * i);
        *len = FbTable::rd<int64_t>(bufs + 16 * i + 8);
        AURON_CHECK(off >= 0 && *len >= 0 && off <= body_len && *len <= body_len - off, "list ScalarValue: buffer outside the body");
        return body + off;
    };
    int64_t l;
    const uint8_t* loffs = buf(1, &l);
    AURON_CHECK(l >= 8, "list ScalarValue: missing list offsets");
    const int32_t first = FbTable::rd<int32_t>(loffs), last = FbTable::rd<int32_t>(loffs + 4);
    const int64_t child_len = FbTable::rd<int64_t>(nodes + 16), child_nulls = FbTable::rd<int64_t>(nodes + 24);
    AURON_CHECK(first >= 0 && last >= first && last <= child_len, "list ScalarValue: bad list offsets");
    out.len = last - first;
    int64_t vl;
    const uint8_t* cv = buf(2, &vl);
    AURON_CHECK(child_len >= 0 && child_len <= (int64_t)INT32_MAX, "list ScalarValue: bad child length");
    if (child_nulls > 0 && vl > 0) {
        AURON_CHECK(vl >= ((int64_t)last + 7) / 8, "list ScalarValue: short validity buffer");
        out.validity.assign((size_t)((out.len + 7) / 8), 0);
        for (int64_t i = 0; i < out.len; i++)
            if ((cv[(first + i) >> 3] >> ((first + i) & 7)) & 1) out.validity[(size_t)(i >> 3)] |= (uint8_t)(1u << (i & 7));
    }
    if (out.type.is_varlen()) {
        int64_t ol, dl;
        const uint8_t* co = buf(3, &ol);
        const uint8_t* cd = buf(4, &dl);
        AURON_CHECK(ol >= (child_len + 1) * 4, "list ScalarValue: short offsets buffer");
        const int32_t b0 = FbTable::rd<int32_t>(co + 4 * (size_t)first);
        out.offsets.resize((size_t)out.len + 1);
        AURON_CHECK(b0 >= 0 && b0 <= dl, "list ScalarValue: string data outside the buffer");
        for (int64_t i = 0; i <= out.len; i++) {
            const int32_t o = FbTable::rd<int32_t>(co + 4 * (size_t)(first + i));
            AURON_CHECK(o >= b0 && o <= dl && (i == 0 || o - b0 >= out.offsets[(size_t)i - 1]), "list ScalarValue: string offsets are not monotonic inside the data buffer");
            out.offsets[(size_t)i] = o - b0;
        }
        out.data.assign(cd + b0, cd + b0 + out.offsets.back());
    } else if (out.type.id == T_BOOL) {
        int64_t dl;
        const uint8_t* cd = buf(3, &dl);
        AURON_CHECK(dl >= ((int64_t)last + 7) / 8, "list ScalarValue: short boolean data buffer");
        out.data.assign((size_t)((out.len + 7) / 8), 0);
        for (int64_t i = 0; i < out.len; i++)
            if ((cd[(first + i) >> 3] >> ((first + i) & 7)) & 1) out.data[(size_t)(i >> 3)] |= (uint8_t)(1u << (i & 7));
    } else if (out.type.id != T_NULL) {
        int64_t dl;
        const uint8_t* cd = buf(3, &dl);
        const int w = out.type.width();
        AURON_CHECK(dl >= (int64_t)last * w, "list ScalarValue: short data buffer");
        out.data.assign(cd + (size_t)first * w, cd + (size_t)last * w);
    }
    return out;
}

bool is_list_scalar_ipc(const uint8_t* bytes, size_t n) {
    const uint8_t* p = bytes;
    const uint8_t *meta, *body;
    uint32_t meta_len;
    int64_t body_len;
    if (!next_ipc_message(p, bytes + n, &meta, &meta_len, &body, &body_len)) return false;
    FbTable msg = FbTable::root(meta, meta_len);
    if (msg.scalar<uint8_t>(1, 0) != 1) return false;
    FbTable schema = msg.table(2);
    if (!schema.ok()) return false;
    uint32_t nfields;
    const uint8_t* fields = schema.vec(1, &nfields);
    if (nfields != 1) return false;
    return schema.vec_table(fields, 0).scalar<uint8_t>(2, 0) == 12;
}

ColumnPtr host_array_to_device(Ctx& ctx, const HostArray& a) {
    auto c = std::make_shared<Column>();
    c->type = a.type;
    c->len = a.len;
    if (!a.validity.empty()) {
        std::vector<uint8_t> v((size_t)bitmap_alloc_bytes(a.len), 0);
        memcpy(v.data(), a.validity.data(), std::min(v.size(), a.validity.size()));
        c->validity = to_device(ctx, v.data(), v.size());
        c->null_count = -1;
    }
    if (a.type.is_varlen()) {
        c->offsets = to_device(ctx, a.offsets.data(), a.offsets.size() * 4);
        c->data = to_device(ctx, a.data.empty() ? (const void*)"" : (const void*)a.data.data(), a.data.size());
        c->data_bytes = (int64_t)a.data.size();
    } else if (a.type.id == T_BOOL) {
        std::vector<uint8_t> v((size_t)bitmap_alloc_bytes(a.len), 0);
        memcpy(v.data(), a.data.data(), std::min(v.size(), a.data.size()));
        c->data = to_device(ctx, v.data(), v.size());
    } else {
        c->data = to_device(ctx, a.data.empty() ? (const void*)"" : (const void*)a.data.data(), a.data.size());
    }
    ctx.sync();
    return c;
}

Literal decode_scalar_ipc(const uint8_t* bytes, size_t n) {
    const uint8_t* p = bytes;
    const uint8_t* end = bytes + n;
    const uint8_t *meta, *body;
    uint32_t meta_len;
    int64_t body_len;
    Literal lit;
    AURON_CHECK(next_ipc_message(p, end, &meta, &meta_len, &body, &body_len), "ScalarValue: missing schema message");
    FbTable msg = FbTable::root(meta, meta_len);
    AURON_CHECK(msg.scalar<uint8_t>(1, 0) == 1, "ScalarValue: first IPC message is not a Schema");
    FbTable schema = msg.table(2);
    AURON_CHECK(schema.ok(), "ScalarValue: Schema message without a header");
    uint32_t nfields;
    const uint8_t* fields = schema.vec(1, &nfields);
    AURON_CHECK(nfields == 1, "ScalarValue: expected exactly one field");
    FbTable field = schema.vec_table(fields, 0);
    lit.type = fb_field_type(field);
    if (!next_ipc_message(p, end, &meta, &meta_len, &body, &body_len)) {
        lit.is_null = true;
        return lit;
    }
    msg = FbTable::root(meta, meta_len);
    AURON_CHECK(msg.scalar<uint8_t>(1, 0) == 3, "ScalarValue: second IPC message is not a RecordBatch");
    FbTable rb = msg.table(2);
    AURON_CHECK(rb.ok(), "ScalarValue: RecordBatch message without a header");
    int64_t length = rb.scalar<int64_t>(0, 0);
    uint32_t nnodes, nbufs;
    const uint8_t* nodes = rb.vec(1, &nnodes, 16);   // FieldNode{length, null_count}
    const uint8_t* bufs = rb.vec(2, &nbufs, 16);     // Buffer{offset, length}
    AURON_CHECK(rb.field_off(3) == 0, "ScalarValue: compressed IPC bodies are not supported");
    if (length == 0 || lit.type.id == T_NULL) {
        lit.is_null = true;
        return lit;
    }
    int64_t null_count = nnodes ? FbTable::rd<int64_t>(nodes + 8) : 0;
    auto buf = [&](uint32_t i, int64_t* len) -> const uint8_t* {
        AURON_CHECK(i < nbufs, "ScalarValue: missing buffer");
        int64_t off = FbTable::rd<int64_t>(bufs + 16 * i);
        *len = FbTable::rd<int64_t>(bufs + 16 * i + 8);
        AURON_CHECK(off >= 0 && *len >= 0 && off <= body_len && *len <= body_len - off, "ScalarValue: buffer outside the body");
        return body + off;
    };
    // the value buffer of a one-row array holds at least one value of the type
    auto value = [&](uint32_t i, int64_t need) -> const uint8_t* {
        int64_t len;
        const uint8_t* p = buf(i, &len);
        AURON_CHECK(len >= need, "ScalarValue: short value buffer");
        return p;
    };
    int64_t vlen;
    const uint8_t* validity = buf(0, &vlen);
    if (null_count > 0 || (vlen > 0 && !(validity[0] & 1))) {   // (buf() checked that vlen bytes exist)
        lit.is_null = true;
        return lit;
    }
    lit.is_null = false;
    switch (lit.type.id) {
        case T_BOOL: lit.i = value(1, 1)[0] & 1; break;
        case T_INT8: lit.i = (int8_t)value(1, 1)[0]; break;
        case T_INT16: lit.i = FbTable::rd<int16_t>(value(1, 2)); break;
        case T_INT32: case T_DATE32: lit.i = FbTable::rd<int32_t>(value(1, 4)); break;
        case T_INT64: case T_DATE64: case T_TIMESTAMP: lit.i = FbTable::rd<int64_t>(value(1, 8)); break;
        case T_FLOAT32: lit.d = FbTable::rd<float>(value(1, 4)); break;
        case T_FLOAT64: lit.d = FbTable::rd<double>(value(1, 8)); break;
        case T_DECIMAL128: {
            const uint8_t* d = value(1, 16);
            lit.lo = FbTable::rd<uint64_t>(d);
            lit.hi = FbTable::rd<int64_t>(d + 8);
            break;
        }
        case T_UTF8: case T_BINARY: {
            const uint8_t* offs = value(1, 8);
            int32_t b0 = FbTable::rd<int32_t>(offs), b1 = FbTable::rd<int32_t>(offs + 4);
            int64_t l2;
            const uint8_t* data = buf(2, &l2);
            AURON_CHECK(b0 >= 0 && b1 >= b0 && b1 <= l2, "ScalarValue: string offsets outside the data buffer");
            lit.s.assign((const char*)data + b0, (size_t)(b1 - b0));
            break;
        }
        default: fail("ScalarValue: unsupported literal type");
    }
    return lit;
}

// ------------------------------------------------------------------------------------------ expressions
static const char* scalar_fn_name(int fun) {   // auron.proto ScalarFunction :213-292
    switch (fun) {
        case 0: return "Abs"; case 1: return "Acos"; case 2: return "Asin"; case 3: return "Atan"; case 4: return "Ascii";
        case 5: return "Ceil"; case 6: return "Cos"; case 8: return "Exp"; case 9: return "Floor"; case 10: return "Ln"; case 11: return "Log";
        case 12: return "Log10"; case 13: return "Log2"; case 14: return "Round"; case 15: return "Signum"; case 16: return "Sin";
        case 17: return "Sqrt"; case 18: return "Tan"; case 19: return "Trunc"; case 20: return "NullIf"; case 22: return "BitLength";
        case 23: return "Btrim"; case 24: return "CharacterLength"; case 25: return "Chr"; case 26: return "Concat"; case 28: return "DatePart";
        case 29: return "DateTrunc"; case 32: return "Lpad"; case 33: return "Lower"; case 34: return "Ltrim"; case 37: return "OctetLength";
        case 41: return "Replace"; case 42: return "Reverse"; case 44: return "Rpad"; case 45: return "Rtrim"; case 51: return "StartsWith";
        case 53: return "Substr"; case 60: return "Translate"; case 61: return "Trim"; case 62: return "Upper"; case 63: return "Coalesce";
        case 64: return "Expm1"; case 65: return "Factorial"; case 66: return "Hex"; case 67: return "Power"; case 68: return "Acosh";
        case 69: return "IsNaN"; case 80: return "Levenshtein"; case 81: return "FindInSet"; case 82: return "Nvl"; case 83: return "Nvl2";
        case 84: return "Least"; case 85: return "Greatest"; case 86: return "MakeDate";
        default: return nullptr;
    }
}

// the plan comes from outside: an expression node with missing operands is an error message, never a null dereference later
static void validate_expr(const Expr& e) {
    for (auto& c : e.children) AURON_CHECK(c != nullptr, "expression node with a missing operand");
    const size_t n = e.children.size();
    switch (e.kind) {
        case E_BINARY: case E_LIKE: case E_SC_AND: case E_SC_OR: AURON_CHECK(n == 2, "expression node needs two operands"); break;
        case E_NOT: case E_IS_NULL: case E_IS_NOT_NULL: case E_NEGATIVE: case E_CAST: case E_TRY_CAST: case E_STARTS_WITH: case E_ENDS_WITH:
        case E_CONTAINS: AURON_CHECK(n == 1, "expression node needs one operand"); break;
        case E_IN_LIST: AURON_CHECK(n >= 1, "IN list without an expression"); break;
        case E_CASE: {
            const size_t extra = (e.has_case_expr ? 1 : 0) + (e.has_else ? 1 : 0);
            AURON_CHECK(n >= extra + 2 && (n - extra) % 2 == 0, "CASE without a complete when/then branch");
            break;
        }
        default: break;
    }
}

static ExprPtr decode_expr_required(const uint8_t* b, size_t n) {
    ExprPtr e = decode_expr(b, n);
    AURON_CHECK(e != nullptr, "Unexpected empty physical expression");
    return e;
}

// nesting guard for the two recursive decoders: a plan nested deeper than any real one is rejected before the stack runs out
static thread_local int g_decode_depth = 0;
struct DepthGuard {
    DepthGuard() {
        AURON_CHECK(g_decode_depth < 2000, "plan nested too deeply");   // (checked before counting: a throwing constructor runs no destructor)
        ++g_decode_depth;
    }
    ~DepthGuard() { --g_decode_depth; }
};
// the partition id of the task whose plan this thread decodes (create_task): the value of SparkPartitionIdExprNode
static thread_local uint32_t g_decode_partition_id = 0;

ExprPtr decode_expr(const uint8_t* b, size_t n) {
    DepthGuard depth;
    PbReader r(b, n);
    uint32_t f, w;
    ExprPtr out;
    while (r.next(&f, &w)) {
        if (w != 2) {
            r.skip(w);
            continue;
        }
        const uint8_t* sb;
        size_t sn;
        r.bytes_view(&sb, &sn);
        auto e = std::make_shared<Expr>();
        PbReader s(sb, sn);
        uint32_t sf, sw;
        auto child = [&](PbReader& rr) {
            const uint8_t* cb;
            size_t cn;
            rr.bytes_view(&cb, &cn);
            return decode_expr_required(cb, cn);
        };
        switch (f) {
            case 1:   // PhysicalColumn{name=1,index=2}: resolved by NAME (planner.rs:855)
                e->kind = E_COLUMN;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) e->name = s.bytes();
                    else s.skip(sw);
                }
                break;
            case 2:   // ScalarValue{ipc_bytes=1}
                e->kind = E_LITERAL;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) {
                        const uint8_t* ib;
                        size_t in;
                        s.bytes_view(&ib, &in);
                        if (is_list_scalar_ipc(ib, in)) {   // a list literal: one list row, broadcast (operators.cc ListExpr)
                            auto h = std::make_shared<HostArray>(decode_list_scalar_ipc(ib, in));
                            e->lit.type = DType::list(h->type, h->elem_nullable, h->elem_name.empty() ? "item" : h->elem_name);
                            e->lit.is_null = h->list_is_null;
                            e->list_lit = h;
                        } else {
                            e->lit = decode_scalar_ipc(ib, in);
                        }
                    } else s.skip(sw);
                }
                break;
            case 3:   // BoundReference{index=1,data_type=2,nullable=3}
                e->kind = E_COLUMN;
                e->index = 0;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 0) e->index = (int)s.varint();
                    else s.skip(sw);
                }
                break;
            case 4:   // PhysicalBinaryExprNode{l=1,r=2,op=3}
                e->kind = E_BINARY;
                e->children.resize(2);
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) e->children[0] = child(s);
                    else if (sf == 2 && sw == 2) e->children[1] = child(s);
                    else if (sf == 3 && sw == 2) e->op = s.bytes();
                    else s.skip(sw);
                }
                AURON_CHECK(e->children[0] && e->children[1], "binary expression missing operand");
                break;
            case 5: fail("Cannot convert aggregate expr node to physical expression");
            case 11: fail("Cannot convert sort expr node to physical expression");
            case 6: case 7: case 8: case 12:
                e->kind = f == 6 ? E_IS_NULL : f == 7 ? E_IS_NOT_NULL : f == 8 ? E_NOT : E_NEGATIVE;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) e->children.push_back(child(s));
                    else s.skip(sw);
                }
                break;
            case 9: {   // PhysicalCaseNode{expr=1, when_then_expr=2{when=1,then=2}, else_expr=3}
                e->kind = E_CASE;
                ExprPtr base, els;
                std::vector<ExprPtr> wt;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) base = child(s);
                    else if (sf == 2 && sw == 2) {
                        const uint8_t* wb;
                        size_t wn;
                        s.bytes_view(&wb, &wn);
                        PbReader wr(wb, wn);
                        uint32_t wf, ww;
                        ExprPtr we, te;
                        while (wr.next(&wf, &ww)) {
                            if (wf == 1 && ww == 2) we = child(wr);
                            else if (wf == 2 && ww == 2) te = child(wr);
                            else wr.skip(ww);
                        }
                        AURON_CHECK(we && te, "CASE branch missing when/then");
                        wt.push_back(we);
                        wt.push_back(te);
                    } else if (sf == 3 && sw == 2) els = child(s);
                    else s.skip(sw);
                }
                if (base) {
                    e->has_case_expr = true;
                    e->children.push_back(base);
                }
                for (auto& x : wt) e->children.push_back(x);
                if (els) {
                    e->has_else = true;
                    e->children.push_back(els);
                }
                break;
            }
            case 10: case 15:   // Cast / TryCast {expr=1, arrow_type=2}
                e->kind = f == 10 ? E_CAST : E_TRY_CAST;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) e->children.push_back(child(s));
                    else if (sf == 2 && sw == 2) {
                        const uint8_t* tb;
                        size_t tn;
                        s.bytes_view(&tb, &tn);
                        e->type = decode_arrow_type(tb, tn);
                    } else s.skip(sw);
                }
                break;
            case 13:   // InList{expr=1, list=2, negated=3}
                e->kind = E_IN_LIST;
                e->children.resize(1);
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) e->children[0] = child(s);
                    else if (sf == 2 && sw == 2) e->children.push_back(child(s));
                    else if (sf == 3 && sw == 0) e->negated = s.varint() != 0;
                    else s.skip(sw);
                }
                break;
            case 14: {   // ScalarFunction{name=1, fun=2, args=3, return_type=4}
                e->kind = E_SCALAR_FN;
                int fun = 0;
                std::string nm;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) nm = s.bytes();
                    else if (sf == 2 && sw == 0) fun = (int)s.varint();
                    else if (sf == 3 && sw == 2) {
                        try {
                            e->children.push_back(child(s));
                        } catch (const Error& err) {   // e.g. an array<string> argument of concat_ws: say which function it was
                            if (makes_string_fn(nm)) fail(nm + ": " + err.what());
                            throw;
                        }
                    } else if (sf == 4 && sw == 2) {
                        const uint8_t* tb;
                        size_t tn;
                        s.bytes_view(&tb, &tn);
                        e->type = decode_arrow_type(tb, tn);
                    } else s.skip(sw);
                }
                if (fun == 10000) e->name = nm;   // AuronExtFunctions: name selects the function (planner.rs:944-960)
                else {
                    const char* k = scalar_fn_name(fun);
                    if (!k) fail("scalar function #" + std::to_string(fun) + " is not native on device");
                    e->name = k;
                }
                break;
            }
            case 20:   // Like{negated=1, case_insensitive=2, expr=3, pattern=4}
                e->kind = E_LIKE;
                e->children.resize(2);
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 0) e->negated = s.varint() != 0;
                    else if (sf == 2 && sw == 0) e->case_insensitive = s.varint() != 0;
                    else if (sf == 3 && sw == 2) e->children[0] = child(s);
                    else if (sf == 4 && sw == 2) e->children[1] = child(s);
                    else s.skip(sw);
                }
                break;
            case 3000: case 3001:
                e->kind = f == 3000 ? E_SC_AND : E_SC_OR;
                e->children.resize(2);
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) e->children[0] = child(s);
                    else if (sf == 2 && sw == 2) e->children[1] = child(s);
                    else s.skip(sw);
                }
                break;
            case 20000: case 20001: case 20002:
                e->kind = f == 20000 ? E_STARTS_WITH : f == 20001 ? E_ENDS_WITH : E_CONTAINS;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) e->children.push_back(child(s));
                    else if (sf == 2 && sw == 2) e->lit.s = s.bytes();
                    else s.skip(sw);
                }
                break;
            case 20100:   // RowNumExprNode{}
                e->kind = E_ROW_NUM;
                break;
            case 20101:   // SparkPartitionIdExprNode{}: the task's partition id, a constant of the plan (spark_partition_id.rs)
                e->kind = E_LITERAL;
                e->lit.type = DType(T_INT32);
                e->lit.is_null = false;
                e->lit.i = (int32_t)g_decode_partition_id;
                break;
            default:
                fail("physical expression kind #" + std::to_string(f) + " is not native on device (JVM-callback / nested-type expressions are out of scope)");
        }
        validate_expr(*e);
        out = e;
    }
    return out;
}

// ------------------------------------------------------------------------------------------ plan nodes
static OperatorPtr decode_plan(Task& t, const uint8_t* b, size_t n);

static OperatorPtr plan_field(Task& t, PbReader& r) {
    const uint8_t* sb;
    size_t sn;
    r.bytes_view(&sb, &sn);
    return decode_plan(t, sb, sn);
}
static ExprPtr expr_field(PbReader& r) {
    const uint8_t* sb;
    size_t sn;
    r.bytes_view(&sb, &sn);
    return decode_expr_required(sb, sn);
}
static Schema schema_field(PbReader& r) {
    const uint8_t* sb;
    size_t sn;
    r.bytes_view(&sb, &sn);
    return decode_schema(sb, sn);
}

static void decode_join_on(PbReader& r, std::vector<ExprPtr>* l, std::vector<ExprPtr>* rr) {
    const uint8_t* sb;
    size_t sn;
    r.bytes_view(&sb, &sn);
    PbReader s(sb, sn);
    uint32_t f, w;
    ExprPtr le, re;
    while (s.next(&f, &w)) {
        if (f == 1 && w == 2) le = expr_field(s);
        else if (f == 2 && w == 2) re = expr_field(s);
        else s.skip(w);
    }
    AURON_CHECK(le && re, "JoinOn needs both sides");
    l->push_back(le);
    rr->push_back(re);
}

SortExprSpec decode_sort_expr(const uint8_t* b, size_t n) {
    // PhysicalExprNode{sort=11{expr=1, asc=2, nulls_first=3}}
    PbReader r(b, n);
    uint32_t f, w;
    SortExprSpec out;
    out.asc = false;
    out.nulls_first = false;
    bool found = false;
    while (r.next(&f, &w)) {
        if (f == 11 && w == 2) {
            const uint8_t* sb;
            size_t sn;
            r.bytes_view(&sb, &sn);
            PbReader s(sb, sn);
            uint32_t sf, sw;
            while (s.next(&sf, &sw)) {
                if (sf == 1 && sw == 2) out.expr = expr_field(s);
                else if (sf == 2 && sw == 0) out.asc = s.varint() != 0;
                else if (sf == 3 && sw == 0) out.nulls_first = s.varint() != 0;
                else s.skip(sw);
            }
            found = true;
        } else r.skip(w);
    }
    AURON_CHECK(found && out.expr, "sort expression expected");
    return out;
}

// list columns pass only through Filter, Project, Limit, Union, Rename, the pass-through nodes, Generate and the Arrow export; the
// operators that sort, hash, serialise or aggregate rows reject a list column they carry or reference when the plan is built
static void reject_list_columns(const char* op, const Schema& s) {
    for (auto& f : s.fields)
        if (f.type.id == T_LIST) fail(std::string(op) + ": list column " + f.name + " (" + f.type.str() + ") is not supported by this operator");
}
static void reject_list_refs(const char* op, const Expr& e, const Schema& s) {
    if (e.kind == E_COLUMN) {
        const int i = e.index >= 0 ? e.index : s.index_of(e.name);
        if (i >= 0 && i < (int)s.fields.size() && s.fields[(size_t)i].type.id == T_LIST)
            fail(std::string(op) + ": list column " + s.fields[(size_t)i].name + " (" + s.fields[(size_t)i].type.str() + ") is not supported by this operator");
    }
    for (auto& c : e.children)
        if (c) reject_list_refs(op, *c, s);
}

static OperatorPtr decode_agg(Task& t, const uint8_t* b, size_t n) {
    PbReader r(b, n);
    uint32_t f, w;
    OperatorPtr input;
    std::vector<ExprPtr> groups;
    std::vector<std::string> gnames, anames;
    std::vector<int> modes;
    std::vector<AggExprSpec> aggs;
    while (r.next(&f, &w)) {
        if (f == 1 && w == 2) input = plan_field(t, r);
        else if (f == 3 && w == 2) groups.push_back(expr_field(r));
        else if (f == 4 && w == 2) {   // PhysicalExprNode{agg_expr=5{agg_function=1, children=3, return_type=4}}
            const uint8_t* sb;
            size_t sn;
            r.bytes_view(&sb, &sn);
            PbReader e(sb, sn);
            uint32_t ef, ew;
            AggExprSpec spec;
            bool found = false;
            while (e.next(&ef, &ew)) {
                if (ef == 5 && ew == 2) {
                    const uint8_t* ab;
                    size_t an;
                    e.bytes_view(&ab, &an);
                    PbReader a(ab, an);
                    uint32_t af, aw;
                    spec.fn = 0;
                    while (a.next(&af, &aw)) {
                        if (af == 1 && aw == 0) spec.fn = (int)a.varint();
                        else if (af == 3 && aw == 2) spec.children.push_back(expr_field(a));
                        else if (af == 4 && aw == 2) {
                            const uint8_t* tb;
                            size_t tn;
                            a.bytes_view(&tb, &tn);
                            spec.return_type = decode_arrow_type(tb, tn);
                        } else a.skip(aw);
                    }
                    found = true;
                } else e.skip(ew);
            }
            AURON_CHECK(found, "Invalid aggregate expression for AggExec");
            aggs.push_back(spec);
        } else if (f == 5 && w == 0) modes.push_back((int)r.varint());
        else if (f == 5 && w == 2) {   // packed repeated enum
            const uint8_t* sb;
            size_t sn;
            r.bytes_view(&sb, &sn);
            PbReader p(sb, sn);
            while (!p.done()) modes.push_back((int)p.varint());
        } else if (f == 6 && w == 2) gnames.push_back(r.bytes());
        else if (f == 7 && w == 2) anames.push_back(r.bytes());
        else r.skip(w);
    }
    AURON_CHECK(input, "AggExecNode without input");
    for (auto& g : groups) reject_list_refs("AggExec", *g, input->out_schema);
    for (auto& a : aggs)
        for (auto& c : a.children) reject_list_refs("AggExec", *c, input->out_schema);
    for (size_t i = 0; i < aggs.size(); i++) {
        aggs[i].mode = i < modes.size() ? modes[i] : MODE_PARTIAL;
        aggs[i].name = i < anames.size() ? anames[i] : "";
    }
    return OperatorPtr(new AggExec(std::move(input), groups, gnames, aggs));
}

static OperatorPtr decode_join(Task& t, const uint8_t* b, size_t n, int kind /*0 hash, 1 smj, 2 broadcast*/) {
    PbReader r(b, n);
    uint32_t f, w;
    Schema schema;
    OperatorPtr left, right;
    std::vector<ExprPtr> lk, rk;
    int jt = JOIN_INNER, side = SIDE_LEFT;   // proto3: a zero-valued enum (LEFT_SIDE = 0) is not on the wire
    bool null_aware = false;
    std::string cache_id;
    std::vector<std::pair<bool, bool>> sort_opts;
    while (r.next(&f, &w)) {
        if (f == 1 && w == 2) schema = schema_field(r);
        else if (f == 2 && w == 2) left = plan_field(t, r);
        else if (f == 3 && w == 2) right = plan_field(t, r);
        else if (f == 4 && w == 2) decode_join_on(r, &lk, &rk);
        else if (kind == 1 && f == 6 && w == 0) jt = (int)r.varint();
        else if (kind == 1 && f == 5 && w == 2) {   // repeated SortOptions{asc=1, nulls_first=2}: one per join key
            const uint8_t* ob;
            size_t on;
            r.bytes_view(&ob, &on);
            PbReader o(ob, on);
            uint32_t of, ow;
            bool asc = false, nf = false;   // proto3 defaults
            while (o.next(&of, &ow)) {
                if (of == 1 && ow == 0) asc = o.varint() != 0;
                else if (of == 2 && ow == 0) nf = o.varint() != 0;
                else o.skip(ow);
            }
            sort_opts.emplace_back(asc, nf);
        }
        else if (kind != 1 && f == 5 && w == 0) jt = (int)r.varint();
        else if (kind != 1 && f == 6 && w == 0) side = (int)r.varint();
        else if (kind == 2 && f == 7 && w == 2) cache_id = r.bytes();
        else if (kind == 2 && f == 8 && w == 0) null_aware = r.varint() != 0;
        else r.skip(w);
    }
    AURON_CHECK(left && right, "join without both inputs");
    const char* jname = kind == 1 ? "SortMergeJoinExec" : kind == 2 ? "BroadcastJoinExec" : "HashJoinExec";
    reject_list_columns(jname, left->out_schema);
    reject_list_columns(jname, right->out_schema);
    reject_list_exprs(lk, left->out_schema, "a join key");
    reject_list_exprs(rk, right->out_schema, "a join key");
    if (kind == 1) return OperatorPtr(new SortMergeJoinExec(std::move(left), std::move(right), lk, rk, sort_opts, jt, schema));
    auto* j = new HashJoinExec(std::move(left), std::move(right), lk, rk, jt, side, schema);
    j->null_aware_anti = null_aware;
    j->cache_id = cache_id;
    return OperatorPtr(j);
}

static OperatorPtr decode_plan(Task& t, const uint8_t* b, size_t n) {
    DepthGuard depth;
    PbReader r(b, n);
    uint32_t f, w;
    OperatorPtr out;
    while (r.next(&f, &w)) {
        if (w != 2) {
            r.skip(w);
            continue;
        }
        const uint8_t* sb;
        size_t sn;
        r.bytes_view(&sb, &sn);
        PbReader s(sb, sn);
        uint32_t sf, sw;
        switch (f) {   // PhysicalPlanNode oneof (auron.proto:27-56)
            case 8: {   // FilterExecNode{input=1, expr=2}  (planner.rs:156-164)
                OperatorPtr input;
                std::vector<ExprPtr> preds;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if (sf == 2 && sw == 2) preds.push_back(expr_field(s));
                    else s.skip(sw);
                }
                AURON_CHECK(input && !preds.empty(), "FilterExecNode needs input and predicates");
                out.reset(new FilterExec(std::move(input), preds));
                break;
            }
            case 6: {   // ProjectionExecNode{input=1, expr=2, expr_name=3, data_type=4}  (planner.rs:130-155)
                OperatorPtr input;
                std::vector<ExprPtr> exprs;
                std::vector<std::string> names;
                std::vector<DType> types;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if (sf == 2 && sw == 2) exprs.push_back(expr_field(s));
                    else if (sf == 3 && sw == 2) names.push_back(s.bytes());
                    else if (sf == 4 && sw == 2) {
                        const uint8_t* tb;
                        size_t tn;
                        s.bytes_view(&tb, &tn);
                        types.push_back(decode_arrow_type(tb, tn));
                    } else s.skip(sw);
                }
                AURON_CHECK(input, "ProjectionExecNode without input");
                out.reset(new ProjectExec(std::move(input), exprs, names, types));
                break;
            }
            case 16: out = decode_agg(t, sb, sn); break;
            case 11: out = decode_join(t, sb, sn, 0); break;
            case 10: out = decode_join(t, sb, sn, 1); break;
            case 13: out = decode_join(t, sb, sn, 2); break;
            case 7: {   // SortExecNode{input=1, expr=2, fetch_limit=3{limit=1, offset=2}}  (planner.rs:355-369)
                OperatorPtr input;
                std::vector<SortExprSpec> keys;
                int64_t limit = -1, offset = 0;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if (sf == 2 && sw == 2) {
                        const uint8_t* eb;
                        size_t en;
                        s.bytes_view(&eb, &en);
                        keys.push_back(decode_sort_expr(eb, en));
                    } else if (sf == 3 && sw == 2) {
                        const uint8_t* lb;
                        size_t ln;
                        s.bytes_view(&lb, &ln);
                        PbReader l(lb, ln);
                        uint32_t lf, lw;
                        limit = 0;
                        while (l.next(&lf, &lw)) {
                            if (lf == 1 && lw == 0) limit = (int64_t)l.varint();
                            else if (lf == 2 && lw == 0) offset = (int64_t)l.varint();
                            else l.skip(lw);
                        }
                    } else s.skip(sw);
                }
                AURON_CHECK(input, "SortExecNode without input");
                reject_list_columns("SortExec", input->out_schema);
                for (auto& k : keys) reject_list_exprs({k.expr}, input->out_schema, "a sort key");
                out.reset(new SortExec(std::move(input), keys, limit, offset));
                break;
            }
            case 17: {   // LimitExecNode{input=1, limit=2, offset=3}
                OperatorPtr input;
                int64_t limit = 0, offset = 0;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if (sf == 2 && sw == 0) limit = (int64_t)s.varint();
                    else if (sf == 3 && sw == 0) offset = (int64_t)s.varint();
                    else s.skip(sw);
                }
                AURON_CHECK(input, "LimitExecNode without input");
                out.reset(new LimitExec(std::move(input), limit, offset));
                break;
            }
            case 18: {   // FFIReaderExecNode{num_partitions=1, schema=2, export_iter_provider_resource_id=3}  (planner.rs:570-577)
                Schema schema;
                std::string id;
                while (s.next(&sf, &sw)) {
                    if (sf == 2 && sw == 2) schema = schema_field(s);
                    else if (sf == 3 && sw == 2) id = s.bytes();
                    else s.skip(sw);
                }
                out.reset(new FFIReaderExec(schema, id));
                break;
            }
            case 3: {   // IpcReaderExecNode{num_partitions=1, schema=2, ipc_provider_resource_id=3}  (planner.rs; auron.proto:636-640)
                Schema schema;
                std::string id;
                while (s.next(&sf, &sw)) {
                    if (sf == 2 && sw == 2) schema = schema_field(s);
                    else if (sf == 3 && sw == 2) id = s.bytes();
                    else s.skip(sw);
                }
                reject_list_columns("IpcReaderExec", schema);
                out = make_ipc_reader(t, schema, id);
                break;
            }
            case 14: {   // RenameColumnsExecNode{input=1, renamed_column_names=2}
                OperatorPtr input;
                std::vector<std::string> names;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if (sf == 2 && sw == 2) names.push_back(s.bytes());
                    else s.skip(sw);
                }
                AURON_CHECK(input, "RenameColumnsExecNode without input");
                out.reset(new RenameColumnsExec(std::move(input), names));
                break;
            }
            case 15: {   // EmptyPartitionsExecNode{schema=1}
                Schema schema;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) schema = schema_field(s);
                    else s.skip(sw);
                }
                out.reset(new EmptyPartitionsExec(schema));
                break;
            }
            case 19: case 12: case 1: {   // CoalesceBatches / BroadcastJoinBuildHashMap / Debug: input = 1
                OperatorPtr input;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else s.skip(sw);
                }
                AURON_CHECK(input, "plan node without input");
                out.reset(new PassThroughExec(std::move(input), f == 19 ? "CoalesceBatchesExec" : f == 12 ? "BroadcastJoinBuildHashMapExec" : "DebugExec"));
                break;
            }
            case 9: {   // UnionExecNode{input=1{input=1, partition=2}, schema=2, num_partitions=3, cur_partition=4}
                std::vector<OperatorPtr> inputs;
                Schema schema;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) {
                        const uint8_t* ub;
                        size_t un;
                        s.bytes_view(&ub, &un);
                        PbReader u(ub, un);
                        uint32_t uf, uw;
                        while (u.next(&uf, &uw)) {
                            if (uf == 1 && uw == 2) inputs.push_back(plan_field(t, u));
                            else u.skip(uw);
                        }
                    } else if (sf == 2 && sw == 2) schema = schema_field(s);
                    else s.skip(sw);
                }
                if (schema.fields.empty() && !inputs.empty()) schema = inputs[0]->out_schema;
                out.reset(new UnionExec(std::move(inputs), schema));
                break;
            }
            case 20: {   // ExpandExecNode{input=1, schema=2, projections=3{expr=1}} (planner.rs:587-602)
                OperatorPtr input;
                Schema schema;
                std::vector<std::vector<std::vector<uint8_t>>> raw;   // expressions are resolved against the input's schema: decoded after it
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if (sf == 2 && sw == 2) schema = schema_field(s);
                    else if (sf == 3 && sw == 2) {
                        const uint8_t* pb;
                        size_t pn;
                        s.bytes_view(&pb, &pn);
                        PbReader pr(pb, pn);
                        uint32_t pf, pw;
                        raw.emplace_back();
                        while (pr.next(&pf, &pw)) {
                            if (pf == 1 && pw == 2) {
                                const uint8_t* eb;
                                size_t en;
                                pr.bytes_view(&eb, &en);
                                raw.back().emplace_back(eb, eb + en);
                            } else pr.skip(pw);
                        }
                    } else s.skip(sw);
                }
                AURON_CHECK(input, "ExpandExecNode without input");
                reject_list_columns("ExpandExec", input->out_schema);
                reject_list_columns("ExpandExec", schema);
                std::vector<std::vector<ExprPtr>> projs;
                for (auto& pr : raw) {
                    projs.emplace_back();
                    for (auto& e : pr) projs.back().push_back(decode_expr(e.data(), e.size()));
                }
                out.reset(new ExpandExec(std::move(input), schema, std::move(projs)));
                break;
            }
            case 22: {   // WindowExecNode{input=1, window_expr=2, partition_spec=3, order_spec=4, group_limit=5{k=1}, output_window_cols=6} (planner.rs:604-760)
                OperatorPtr input;
                std::vector<std::vector<uint8_t>> raw_funcs, raw_part, raw_order;
                int64_t limit = -1;
                bool out_cols = false;   // proto3: an omitted bool is false
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if ((sf == 2 || sf == 3 || sf == 4) && sw == 2) {
                        const uint8_t* eb;
                        size_t en;
                        s.bytes_view(&eb, &en);
                        (sf == 2 ? raw_funcs : sf == 3 ? raw_part : raw_order).emplace_back(eb, eb + en);
                    } else if (sf == 5 && sw == 2) {
                        const uint8_t* lb;
                        size_t ln;
                        s.bytes_view(&lb, &ln);
                        PbReader l(lb, ln);
                        uint32_t lf, lw;
                        limit = 0;
                        while (l.next(&lf, &lw)) {
                            if (lf == 1 && lw == 0) limit = (int64_t)l.varint();
                            else l.skip(lw);
                        }
                    } else if (sf == 6 && sw == 0) out_cols = s.varint() != 0;
                    else s.skip(sw);
                }
                AURON_CHECK(input, "WindowExecNode without input");
                reject_list_columns("WindowExec", input->out_schema);
                std::vector<ExprPtr> part, order;
                for (auto& e : raw_part) part.push_back(decode_expr(e.data(), e.size()));
                for (auto& e : raw_order) order.push_back(decode_sort_expr(e.data(), e.size()).expr);   // (the direction is the sort's business: only equality of neighbours matters here)
                std::vector<WindowFuncSpec> funcs;
                for (auto& wbytes : raw_funcs) {   // WindowExprNode{field=1, return_type=1000, func_type=2, window_func=3, agg_func=4, children=5}
                    PbReader w(wbytes.data(), wbytes.size());
                    uint32_t wf, ww;
                    WindowFuncSpec spec;
                    int func_type = 0, window_func = 0, agg_func = 0;
                    const uint8_t *field_b = nullptr, *type_b = nullptr;
                    size_t field_n = 0, type_n = 0;
                    std::vector<std::pair<const uint8_t*, size_t>> arg_b;
                    while (w.next(&wf, &ww)) {
                        const uint8_t* vb;
                        size_t vn;
                        if (wf == 1 && ww == 2) w.bytes_view(&field_b, &field_n);
                        else if (wf == 1000 && ww == 2) w.bytes_view(&type_b, &type_n);
                        else if (wf == 2 && ww == 0) func_type = (int)w.varint();
                        else if (wf == 3 && ww == 0) window_func = (int)w.varint();
                        else if (wf == 4 && ww == 0) agg_func = (int)w.varint();
                        else if (wf == 5 && ww == 2) {
                            w.bytes_view(&vb, &vn);
                            arg_b.emplace_back(vb, vn);
                        } else w.skip(ww);
                    }
                    spec.is_agg = func_type == 1;
                    spec.func = spec.is_agg ? agg_func : window_func;
                    // types and arguments are decoded once the function is known, so that an unsupported one names it
                    try {
                        if (field_b) spec.field = decode_field(field_b, field_n);
                        if (type_b) spec.field.type = decode_arrow_type(type_b, type_n);   // return_type repeats the field's type
                        if (spec.field.type.id == T_LIST) fail("a list result (" + spec.field.type.str() + ") is not supported");
                        for (auto& a : arg_b) spec.args.push_back(decode_expr(a.first, a.second));
                    } catch (const Error& e) {
                        static const char* wfn[] = {"ROW_NUMBER", "RANK", "DENSE_RANK", "LEAD", "NTH_VALUE", "NTH_VALUE_IGNORE_NULLS", "PERCENT_RANK", "CUME_DIST"};
                        static const char* afn[] = {"MIN", "MAX", "SUM", "AVG", "COUNT"};
                        const int nf = spec.is_agg ? 5 : 8;
                        const std::string fname = spec.func >= 0 && spec.func < nf ? (spec.is_agg ? afn : wfn)[spec.func] : "#" + std::to_string(spec.func);
                        fail("window " + fname + ": " + e.what());
                    }
                    funcs.push_back(std::move(spec));
                }
                reject_list_exprs(part, input->out_schema, "a window partition key");
                reject_list_exprs(order, input->out_schema, "a window order key");
                for (auto& fs : funcs) reject_list_exprs(fs.args, input->out_schema, "a window function argument");
                out.reset(new WindowExec(std::move(input), std::move(part), std::move(order), std::move(funcs), limit, out_cols));
                break;
            }
            case 4: {   // IpcWriterExecNode{input=1, ipc_consumer_resource_id=2}
                OperatorPtr input;
                std::string rid;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if (sf == 2 && sw == 2) rid = s.bytes();
                    else s.skip(sw);
                }
                AURON_CHECK(input, "IpcWriterExecNode without input");
                reject_list_columns("IpcWriterExec", input->out_schema);
                out = make_ipc_writer(t, std::move(input), rid);
                break;
            }
            case 5:
                out = make_parquet_scan(t, sb, sn);   // (reads one-level LIST columns of flat elements; rejects list partition columns)
                break;
            case 23: {   // GenerateExecNode{input=1, generator=2{func=1, udtf=2, child=3}, required_child_output=3, generator_output=4, outer=5}
                OperatorPtr input;
                bool has_gen = false, outer = false, has_udtf = false;
                int func = 0;
                std::vector<std::vector<uint8_t>> raw_child;   // resolved against the input's schema: decoded after it
                std::vector<std::string> req;
                std::vector<Field> gout;
                while (s.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s);
                    else if (sf == 2 && sw == 2) {
                        has_gen = true;
                        const uint8_t* gb;
                        size_t gn;
                        s.bytes_view(&gb, &gn);
                        PbReader g(gb, gn);
                        uint32_t gf, gw;
                        while (g.next(&gf, &gw)) {
                            if (gf == 1 && gw == 0) func = (int)g.varint();
                            else if (gf == 2 && gw == 2) {
                                has_udtf = true;
                                g.skip(gw);
                            } else if (gf == 3 && gw == 2) {
                                const uint8_t* cb;
                                size_t cn;
                                g.bytes_view(&cb, &cn);
                                raw_child.emplace_back(cb, cb + cn);
                            } else g.skip(gw);
                        }
                    } else if (sf == 3 && sw == 2) req.push_back(s.bytes());
                    else if (sf == 4 && sw == 2) {
                        const uint8_t* fb;
                        size_t fn;
                        s.bytes_view(&fb, &fn);
                        gout.push_back(decode_field(fb, fn));
                    } else if (sf == 5 && sw == 0) outer = s.varint() != 0;
                    else s.skip(sw);
                }
                AURON_CHECK(input, "GenerateExecNode without input");
                if (!has_gen) fail("GenerateExec without a generator is not native in auron_b200");
                if (func == 2) fail("generate function JsonTuple is not native in auron_b200");
                if (func == 10000 || has_udtf) fail("generate function Udtf is not native in auron_b200");
                if (func != GEN_EXPLODE && func != GEN_POS_EXPLODE) fail("generate function #" + std::to_string(func) + " is not native in auron_b200");
                if (raw_child.size() != 1) fail(std::string(func == GEN_POS_EXPLODE ? "PosExplode" : "Explode") + " takes one child expression, got " + std::to_string(raw_child.size()));
                ExprPtr child = decode_expr_required(raw_child[0].data(), raw_child[0].size());
                out.reset(new GenerateExec(std::move(input), func, child, std::move(req), std::move(gout), outer));
                break;
            }
            case 2: {   // ShuffleWriterExecNode{input=1, ...}
                OperatorPtr input;
                PbReader s2(sb, sn);
                while (s2.next(&sf, &sw)) {
                    if (sf == 1 && sw == 2) input = plan_field(t, s2);
                    else s2.skip(sw);
                }
                AURON_CHECK(input, "ShuffleWriterExecNode without input");
                reject_list_columns("ShuffleWriterExec", input->out_schema);
                out = make_shuffle_writer(t, std::move(input), sb, sn);
                break;
            }
            default:
                fail("plan node #" + std::to_string(f) + " is not native in auron_b200 (see DESIGN.md scope)");
        }
    }
    AURON_CHECK(out != nullptr, "empty PhysicalPlanNode");
    return out;
}

std::unique_ptr<Task> create_task(const uint8_t* task_def, size_t len, const auron_callbacks* cb, int device) {
    auto t = std::make_unique<Task>(device);
    t->cb = cb;
    PbReader r(task_def, len);
    uint32_t f, w;
    const uint8_t* plan = nullptr;
    size_t plan_len = 0;
    while (r.next(&f, &w)) {
        if (f == 1 && w == 2) {   // PartitionId{stage_id=2, partition_id=4, task_id=5}
            const uint8_t* sb;
            size_t sn;
            r.bytes_view(&sb, &sn);
            PbReader s(sb, sn);
            uint32_t sf, sw;
            while (s.next(&sf, &sw)) {
                if (sf == 2 && sw == 0) t->stage_id = (uint32_t)s.varint();
                else if (sf == 4 && sw == 0) t->partition_id = (uint32_t)s.varint();
                else if (sf == 5 && sw == 0) t->task_id = s.varint();
                else s.skip(sw);
            }
        } else if (f == 2 && w == 2) r.bytes_view(&plan, &plan_len);   // decoded once the partition id is known
        else r.skip(w);
    }
    if (plan) {
        g_decode_partition_id = t->partition_id;
        t->root = decode_plan(*t, plan, plan_len);
    }
    AURON_CHECK(t->root != nullptr, "TaskDefinition without a plan");
    return t;
}

}  // namespace auron
