// operators.cc -- operator implementations (see operators.h for the reference files they mirror).
// Every operator works on large device-resident chunks; the 10,000-row batch size of the reference
// (datafusion-ext-commons/src/lib.rs:72-75) only survives as the JVM-facing default and is not part of
// the result contract (SURVEY.md Appendix B.2).
#include "operators.h"
#include "mem_manager.h"

#include <algorithm>
#include <map>
#include <mutex>

#include "../../include/auron_b200.h"

namespace auron {

bool Task::is_running() {
    if (cancelled) return false;
    if (cb && cb->is_task_running) return cb->is_task_running(cb->user) != 0;
    return true;
}

std::string Task::conf(const char* key, const char* env, const char* dflt) const {
    if (cb && cb->get_conf) {
        char buf[256];
        int n = cb->get_conf(cb->user, key, buf, (int32_t)sizeof(buf));
        if (n >= 0 && n < (int)sizeof(buf)) return std::string(buf, (size_t)n);
    }
    if (env)
        if (const char* e = getenv(env)) return e;
    return dflt ? dflt : "";
}

// ------------------------------------------------------------------------------------------ explain
std::string json_quote(const std::string& s) {
    std::string o = "\"";
    for (char c : s) {
        if (c == '"' || c == '\\') o.push_back('\\');
        if ((unsigned char)c < 0x20) o += ' ';
        else o.push_back(c);
    }
    return o + "\"";
}
static std::string lit_to_string(const Literal& l) {
    if (l.is_null) return "lit(" + l.type.str() + ":NULL)";
    if (l.type.id == T_LIST) return "lit(" + l.type.str() + ")";
    std::string v;
    switch (l.type.id) {
        case T_FLOAT32: case T_FLOAT64: {
            char buf[64];
            snprintf(buf, sizeof(buf), "%.17g", l.d);
            v = buf;
            break;
        }
        case T_UTF8: case T_BINARY: v = "'" + l.s + "'"; break;
        case T_DECIMAL128: {   // unscaled value
            unsigned __int128 mag = ((unsigned __int128)(uint64_t)l.hi << 64) | l.lo;
            const bool neg = l.hi < 0;
            if (neg) mag = ~mag + 1;
            std::string d;
            do {
                d.insert(d.begin(), (char)('0' + (int)(mag % 10)));
                mag /= 10;
            } while (mag);
            v = (neg ? "-" : "") + d;
            break;
        }
        default: v = std::to_string(l.i);
    }
    return "lit(" + l.type.str() + ":" + v + ")";
}
std::string expr_to_string(const Expr& e) {
    auto args = [&](size_t from = 0) {
        std::string a;
        for (size_t i = from; i < e.children.size(); i++) a += (i > from ? ", " : "") + expr_to_string(*e.children[i]);
        return a;
    };
    switch (e.kind) {
        case E_COLUMN: return e.index >= 0 ? "col(#" + std::to_string(e.index) + ")" : "col(" + e.name + ")";
        case E_LITERAL: return lit_to_string(e.lit);
        case E_BINARY: return e.op + "(" + args() + ")";
        case E_NOT: return "Not(" + args() + ")";
        case E_IS_NULL: return "IsNull(" + args() + ")";
        case E_IS_NOT_NULL: return "IsNotNull(" + args() + ")";
        case E_NEGATIVE: return "Negative(" + args() + ")";
        case E_CASE: return std::string("Case") + (e.has_case_expr ? "[expr]" : "") + (e.has_else ? "[else]" : "") + "(" + args() + ")";
        case E_CAST: return "Cast(" + args() + " AS " + e.type.str() + ")";
        case E_TRY_CAST: return "TryCast(" + args() + " AS " + e.type.str() + ")";
        case E_IN_LIST: return std::string(e.negated ? "NotIn(" : "In(") + args() + ")";
        case E_SCALAR_FN: return e.name + "(" + args() + ") -> " + e.type.str();
        case E_LIKE: return std::string(e.negated ? "NotLike" : "Like") + (e.case_insensitive ? "[i](" : "(") + args() + ")";
        case E_STARTS_WITH: return "StartsWith(" + args() + ", '" + e.lit.s + "')";
        case E_ENDS_WITH: return "EndsWith(" + args() + ", '" + e.lit.s + "')";
        case E_CONTAINS: return "Contains(" + args() + ", '" + e.lit.s + "')";
        case E_SC_AND: return "SCAnd(" + args() + ")";
        case E_SC_OR: return "SCOr(" + args() + ")";
        case E_ROW_NUM: return "RowNum()";
    }
    return "?";
}
static std::string exprs_json(const std::vector<ExprPtr>& es) {
    std::string o = "[";
    for (size_t i = 0; i < es.size(); i++) o += (i ? "," : "") + json_quote(expr_to_string(*es[i]));
    return o + "]";
}

std::string FFIReaderExec::describe() const { return "\"resource_id\":" + json_quote(resource_id); }
std::string FilterExec::describe() const { return "\"predicates\":" + exprs_json(predicates); }
std::string ProjectExec::describe() const { return "\"exprs\":" + exprs_json(exprs); }
std::string GenerateExec::describe() const {
    std::string o = std::string("\"function\":\"") + (func == GEN_POS_EXPLODE ? "PosExplode" : "Explode") + "\",\"outer\":" + (outer ? "true" : "false") +
                    ",\"child\":" + json_quote(gen.text) + ",\"required\":[";
    for (size_t i = 0; i < required_names.size(); i++) o += (i ? "," : "") + json_quote(required_names[i]);
    o += "],\"generator_output\":[";
    for (size_t i = 0; i < gen_fields.size(); i++) o += std::string(i ? "," : "") + "[" + json_quote(gen_fields[i].name) + "," + json_quote(gen_fields[i].type.str()) + "]";
    return o + "]";
}
std::string AggExec::describe() const {
    static const char* fn_names[] = {"MIN", "MAX", "SUM", "AVG", "COUNT", "?", "?", "FIRST", "FIRST_IGNORES_NULL"};
    static const char* mode_names[] = {"PARTIAL", "PARTIAL_MERGE", "FINAL"};
    std::string o = "\"grouping\":" + exprs_json(group_exprs) + ",\"aggs\":[";
    for (size_t i = 0; i < aggs.size(); i++) {
        const auto& a = aggs[i];
        o += std::string(i ? "," : "") + "{\"fn\":\"" + (a.fn >= 0 && a.fn <= 8 ? fn_names[a.fn] : "?") + "\",\"mode\":\"" +
             (a.mode >= 0 && a.mode <= 2 ? mode_names[a.mode] : "?") + "\",\"args\":" + exprs_json(a.children) + ",\"return_type\":" + json_quote(a.return_type.str()) + "}";
    }
    return o + "]";
}
std::string HashJoinExec::describe() const {
    static const char* jt[] = {"INNER", "LEFT", "RIGHT", "FULL", "SEMI", "ANTI", "EXISTENCE"};
    return std::string("\"join_type\":\"") + (join_type >= 0 && join_type <= 6 ? jt[join_type] : "?") + "\",\"build_side\":\"" +
           (build_side == SIDE_LEFT ? "LEFT" : "RIGHT") + "\",\"left_keys\":" + exprs_json(left_keys) + ",\"right_keys\":" + exprs_json(right_keys) +
           ",\"cached_build_hash_map_id\":" + json_quote(cache_id) + ",\"null_aware_anti\":" + (null_aware_anti ? "true" : "false");
}
std::string SortExec::describe() const {
    std::string o = "\"keys\":[";
    for (size_t i = 0; i < keys.size(); i++)
        o += (i ? "," : "") + json_quote(expr_to_string(*keys[i].expr) + (keys[i].asc ? " ASC" : " DESC") + (keys[i].nulls_first ? " NULLS FIRST" : " NULLS LAST"));
    return o + "],\"limit\":" + std::to_string(limit) + ",\"offset\":" + std::to_string(offset);
}
std::string LimitExec::describe() const { return "\"limit\":" + std::to_string(limit) + ",\"offset\":" + std::to_string(offset); }

// ------------------------------------------------------------------------------------------ resources
struct DevResource {
    std::vector<BatchPtr> batches;
    Schema schema;
};
static std::mutex g_res_mu;
static std::map<std::string, DevResource> g_resources;
void put_device_resource(const std::string& id, std::vector<BatchPtr> batches, const Schema& schema) {
    std::lock_guard<std::mutex> l(g_res_mu);
    auto& r = g_resources[id];
    r.schema = schema;
    for (auto& b : batches) r.batches.push_back(b);
}
bool get_device_resource(const std::string& id, std::vector<BatchPtr>* batches, Schema* schema) {
    std::lock_guard<std::mutex> l(g_res_mu);
    auto it = g_resources.find(id);
    if (it == g_resources.end()) return false;
    if (batches) *batches = it->second.batches;
    if (schema) *schema = it->second.schema;
    return true;
}
void drop_device_resource(const std::string& id) {
    std::lock_guard<std::mutex> l(g_res_mu);
    g_resources.erase(id);
}

const int32_t* ensure_sel(Task& t, SelBatch& s) {
    if (!s.sel && s.mask && s.batch) {
        int64_t cnt = 0;
        s.sel = mask_to_indices(t.ctx, P<uint32_t>(s.mask), s.batch->num_rows, &cnt);
        s.n = cnt;
        s.mask.reset();
    }
    return P<int32_t>(s.sel);
}
BatchPtr materialize(Task& t, SelBatch& s) {
    if (!s.batch) return nullptr;
    const int32_t* sel = ensure_sel(t, s);
    if (!sel) return s.batch;
    return take_batch(t.ctx, *s.batch, sel, s.n, false);
}

ColumnPtr eval_to_column(Task& t, const ExprPtr& e, const Schema& schema, const Batch& b) {
    int idx;
    if (is_plain_column(*e, schema, &idx)) return b.cols[idx];
    VmProgram p = compile_projection({e}, schema);
    return eval_projection(t.ctx, p, b, nullptr, b.num_rows)[0];
}

// ------------------------------------------------------------------------------------------ FFIReaderExec
FFIReaderExec::FFIReaderExec(const Schema& schema, const std::string& id) : resource_id(id) {
    name = "FFIReaderExec";
    out_schema = schema;
    Schema rs;
    if (get_device_resource(id, &dev_batches, &rs)) {
        is_device = true;
        AURON_CHECK(rs.fields.size() == schema.fields.size(), "device resource schema mismatch for " + id);
    }
}
BatchPtr FFIReaderExec::next(Task& t) {
    if (done) return nullptr;
    if (is_device) {
        if (dev_pos >= dev_batches.size()) {
            done = true;
            return nullptr;
        }
        auto b = dev_batches[dev_pos++];
        metrics.add("output_rows", b->num_rows);
        return b;
    }
    AURON_CHECK(t.cb && t.cb->export_next_batch, "FFIReaderExec needs the export_next_batch callback");
    std::vector<BatchPtr> got;
    int64_t rows = 0;
    while (rows < t.ctx.gpu_chunk_rows) {
        ArrowArray arr;
        memset(&arr, 0, sizeof(arr));
        int rc = t.cb->export_next_batch(t.cb->user, resource_id.c_str(), &arr);
        if (rc < 0) fail("export_next_batch failed for resource " + resource_id);
        if (rc == 0) {
            done = true;
            break;
        }
        BatchPtr b;
        try {
            b = import_batch(t.ctx, &arr, out_schema);
        } catch (...) {
            if (arr.release) arr.release(&arr);
            throw;
        }
        if (arr.release) arr.release(&arr);   // engine owns the exported array (ffi_reader_exec.rs:182-251)
        rows += b->num_rows;
        if (b->num_rows) got.push_back(b);
    }
    if (got.empty()) return nullptr;
    metrics.add("output_rows", rows);
    return concat_batches(t.ctx, got);
}

// ------------------------------------------------------------------------------------------ FilterExec
FilterExec::FilterExec(OperatorPtr input, std::vector<ExprPtr> preds) : predicates(std::move(preds)) {
    name = "FilterExec";
    out_schema = input->out_schema;
    children.push_back(std::move(input));
    prog = compile_predicate(predicates, out_schema);
}
SelBatch FilterExec::next_sel(Task& t) {
    BatchPtr b = children[0]->next(t);
    if (!b) return SelBatch();
    return apply(t, b);
}
SelBatch FilterExec::apply(Task& t, const BatchPtr& b) {
    SelBatch out;
    OpTimer timer(metrics, "elapsed_ns");
    out.batch = b;
    // the selection stays a bit mask until a consumer needs row indices (ensure_sel): Filter -> HashAggregate never does
    Buf mask = eval_predicate(t.ctx, prog, *b, b->num_rows);
    int64_t cnt = count_set_bits(t.ctx, (const uint8_t*)mask->ptr, b->num_rows);
    out.n = cnt;
    if (cnt != b->num_rows) out.mask = mask;
    metrics.add("output_rows", cnt);
    return out;
}
BatchPtr FilterExec::next(Task& t) {
    SelBatch s = next_sel(t);
    return materialize(t, s);
}

// ------------------------------------------------------------------------------------------ ProjectExec
ProjectExec::ProjectExec(OperatorPtr input, std::vector<ExprPtr> ex, std::vector<std::string> names, std::vector<DType> types)
    : exprs(std::move(ex)) {
    name = "ProjectExec";
    const Schema& in = input->out_schema;
    std::vector<ExprPtr> computed;
    for (size_t i = 0; i < exprs.size(); i++) {
        DType actual = infer_type(*exprs[i], in);
        DType declared = i < types.size() && types[i].id != T_NULL ? types[i] : actual;
        const std::string fname = i < names.size() ? names[i] : ("c" + std::to_string(i));
        if (actual.id == T_LIST || declared.id == T_LIST) {   // a list value: a bare column, or computed after the VM
            if (actual != declared) fail("ProjectExec: " + fname + " is " + actual.str() + " but declared " + declared.str() + ": a cast of a list is not supported");
            int idx = -1;
            ListExpr le;
            if (is_plain_column(*exprs[i], in, &idx)) {
                plain_col.push_back(idx);
                list_slot.push_back(-1);
            } else {
                plan_list_expr(exprs[i], in, declared, &le, &computed);
                plain_col.push_back(-1);
                list_slot.push_back((int)lists.size());
                lists.push_back(std::move(le));
            }
            prog_slot.push_back(-1);
            out_schema.fields.push_back(Field{fname, declared, true});
            continue;
        }
        list_slot.push_back(-1);
        if (actual != declared) {   // planner.rs:145-149 wraps a TryCastExpr when the declared type differs
            auto c = std::make_shared<Expr>();
            c->kind = E_TRY_CAST;
            c->type = declared;
            c->children.push_back(exprs[i]);
            exprs[i] = c;
        }
        int idx = -1;
        if (is_plain_column(*exprs[i], in, &idx)) {
            plain_col.push_back(idx);
            prog_slot.push_back(-1);
        } else {
            plain_col.push_back(-1);
            prog_slot.push_back((int)computed.size());
            computed.push_back(exprs[i]);
        }
        Field f;
        f.name = fname;
        f.type = declared;
        out_schema.fields.push_back(f);
    }
    if (!computed.empty()) {
        prog = compile_projection(computed, in, true);
        has_prog = true;
    }
    children.push_back(std::move(input));
}
BatchPtr ProjectExec::next(Task& t) {
    SelBatch s = children[0]->next_sel(t);
    if (!s.batch) return nullptr;
    ensure_sel(t, s);
    auto out = std::make_shared<Batch>();
    out->num_rows = s.n;
    std::vector<ColumnPtr> computed;
    if (has_prog) computed = eval_projection(t.ctx, prog, *s.batch, P<int32_t>(s.sel), s.n, rows_out);
    rows_out += s.n;
    for (size_t i = 0; i < exprs.size(); i++) {
        if (plain_col[i] >= 0) {
            const ColumnPtr& c = s.batch->cols[plain_col[i]];
            out->cols.push_back(s.sel ? take(t.ctx, *c, P<int32_t>(s.sel), s.n, false) : c);
        } else if (list_slot[i] >= 0) {
            out->cols.push_back(eval_list_expr(t, lists[(size_t)list_slot[i]], *s.batch, P<int32_t>(s.sel), s.n, computed));
        } else {
            out->cols.push_back(computed[prog_slot[i]]);
        }
    }
    metrics.add("output_rows", s.n);
    return out;
}

// ------------------------------------------------------------------------------------------ list expressions
bool plan_list_expr(const ExprPtr& e, const Schema& in, const DType& declared, ListExpr* out, std::vector<ExprPtr>* args) {
    const DType actual = infer_type(*e, in);
    if (actual.id != T_LIST) return false;
    out->type = declared.id == T_LIST ? declared : actual;
    out->text = expr_to_string(*e);
    int idx = -1;
    if (is_plain_column(*e, in, &idx)) {
        out->kind = ListExpr::COLUMN;
        out->col = idx;
        return true;
    }
    if (e->kind == E_LITERAL) {
        out->kind = ListExpr::LITERAL;
        out->lit = e->list_lit;
        AURON_CHECK(out->lit != nullptr, "list literal without its elements");
        return true;
    }
    if (e->kind == E_SCALAR_FN && e->name == "Spark_StringSplit") {   // spark_strings.rs:93-115 (ShimsImpl: split(s, <literal>))
        if (e->children.size() != 2) fail("Spark_StringSplit takes a string and a pattern");
        const Expr& pat = *e->children[1];
        if (pat.kind != E_LITERAL || pat.lit.type.id != T_UTF8 || pat.lit.is_null || pat.lit.s.empty())
            fail("Spark_StringSplit: the pattern must be a non-empty utf8 literal, got " + expr_to_string(pat));
        const DType st = infer_type(*e->children[0], in);
        if (st.id != T_UTF8) fail("Spark_StringSplit needs a utf8 string, got " + st.str());
        out->kind = ListExpr::SPLIT;
        out->pattern = pat.lit.s;
        out->arg_slots.push_back((int)args->size());
        args->push_back(e->children[0]);
        return true;
    }
    if (e->kind == E_SCALAR_FN && e->name == "Spark_MakeArray") {   // spark_make_array.rs
        if (e->children.empty()) fail("Spark_MakeArray needs at least one argument");
        const DType et = infer_type(*e->children[0], in);
        for (auto& c : e->children) {
            const DType ct = infer_type(*c, in);
            if (ct != et || ct.id == T_NULL || ct.id == T_LIST)
                fail("Spark_MakeArray: every argument must have one flat type, got " + et.str() + " and " + ct.str());
        }
        out->kind = ListExpr::MAKE_ARRAY;
        for (auto& c : e->children) {
            out->arg_slots.push_back((int)args->size());
            args->push_back(c);
        }
        return true;
    }
    fail(expr_to_string(*e) + ": this list expression is not native on device (only list columns, list literals, Spark_StringSplit and Spark_MakeArray)");
}
ColumnPtr eval_list_expr(Task& t, ListExpr& le, const Batch& b, const int32_t* sel, int64_t n, const std::vector<ColumnPtr>& computed) {
    switch (le.kind) {
        case ListExpr::COLUMN: {
            const ColumnPtr& c = b.cols[(size_t)le.col];
            return sel ? take(t.ctx, *c, sel, n, false) : c;
        }
        case ListExpr::LITERAL:
            if (!le.lit_dev) le.lit_dev = host_array_to_device(t.ctx, *le.lit);
            return broadcast_list(t.ctx, le.lit_dev, le.lit->list_is_null, n, le.type);
        case ListExpr::SPLIT: return string_split(t.ctx, *computed[(size_t)le.arg_slots[0]], le.pattern, le.type);
        case ListExpr::MAKE_ARRAY: {
            std::vector<ColumnPtr> args;
            for (int k : le.arg_slots) args.push_back(computed[(size_t)k]);
            return make_array(t.ctx, args, n, le.type);
        }
    }
    fail("unknown list expression");
}

// ------------------------------------------------------------------------------------------ GenerateExec
GenerateExec::GenerateExec(OperatorPtr input, int fn, const ExprPtr& child, std::vector<std::string> req, std::vector<Field> gen_output, bool out)
    : func(fn), outer(out), required_names(std::move(req)), gen_fields(std::move(gen_output)) {
    name = "GenerateExec";
    const Schema& in = input->out_schema;
    const char* fname = func == GEN_POS_EXPLODE ? "PosExplode" : "Explode";
    std::vector<ExprPtr> args;
    const DType ct = infer_type(*child, in);
    if (ct.id != T_LIST) fail(std::string(fname) + " of a " + ct.str() + " value is not native in auron_b200 (only lists are exploded)");
    plan_list_expr(child, in, ct, &gen, &args);
    if (!args.empty()) {
        prog = compile_projection(args, in);
        has_prog = true;
    }
    for (auto& nm : required_names) {   // planner.rs:790-795: resolved by name
        const int i = in.index_of(nm);
        if (i < 0) fail("GenerateExec: required child column " + nm + " is not in the input schema");
        required.push_back(i);
        out_schema.fields.push_back(in.fields[(size_t)i]);
    }
    // generator output: [pos int32,] element, of exactly the types the generator produces (Spark always sends them so)
    const size_t want = func == GEN_POS_EXPLODE ? 2 : 1;
    if (gen_fields.size() != want) fail(std::string("GenerateExec: ") + fname + " produces " + std::to_string(want) + " columns, the plan declares " + std::to_string(gen_fields.size()));
    if (func == GEN_POS_EXPLODE && gen_fields[0].type != DType(T_INT32))
        fail("GenerateExec: PosExplode's position column " + gen_fields[0].name + " must be int32, the plan declares " + gen_fields[0].type.str());
    const Field& ef = gen_fields.back();
    if (ef.type != *gen.type.elem)
        fail("GenerateExec: " + std::string(fname) + "'s value column " + ef.name + " must be " + gen.type.elem->str() + ", the plan declares " + ef.type.str());
    for (auto& f : gen_fields) out_schema.fields.push_back(f);
    children.push_back(std::move(input));
}
BatchPtr GenerateExec::next(Task& t) {
    for (;;) {
        if (!cur.batch || next_row >= cur.n) {
            cur = children[0]->next_sel(t);
            if (!cur.batch) return nullptr;
            OpTimer timer(metrics, "elapsed_compute");
            const int32_t* sel = ensure_sel(t, cur);
            std::vector<ColumnPtr> computed;
            if (has_prog) computed = eval_projection(t.ctx, prog, *cur.batch, sel, cur.n);
            list = eval_list_expr(t, gen, *cur.batch, sel, cur.n, computed);
            std::vector<ColumnPtr> var;
            for (int c : required)
                if (cur.batch->cols[(size_t)c]->type.is_varlen()) var.push_back(cur.batch->cols[(size_t)c]);
            explode_scan(t.ctx, *list, outer, var, sel, cur.n, &rows_cum, &bytes_cum);
            next_row = 0;
            if (cur.n == 0) continue;
        }
        OpTimer timer(metrics, "elapsed_compute");
        const int64_t r0 = next_row;
        int64_t rows = 0, bytes = 0;
        const int64_t r1 = explode_cut(t.ctx, rows_cum, bytes_cum, cur.n, r0, t.ctx.gpu_chunk_rows, (int64_t)INT32_MAX, &rows, &bytes);
        next_row = r1;
        if (bytes > (int64_t)INT32_MAX)
            fail("GenerateExec: input row " + std::to_string(r0) + " explodes into " + std::to_string(bytes) +
                 " bytes of required string columns, more than int32 offsets address in one batch");
        if (rows > (int64_t)INT32_MAX) fail("GenerateExec: input row " + std::to_string(r0) + " explodes into more than 2^31 - 1 rows");
        if (rows == 0) continue;
        const int32_t* sel = P<int32_t>(cur.sel);
        Buf row_idx = dalloc(t.ctx, (size_t)rows * 4), elem_idx = dalloc(t.ctx, (size_t)rows * 4);
        Buf pos, pos_valid;
        if (func == GEN_POS_EXPLODE) {
            pos = dalloc(t.ctx, (size_t)rows * 4);
            if (outer) pos_valid = dalloc(t.ctx, bitmap_alloc_bytes(rows));
        }
        explode_map(t.ctx, *list, sel, rows_cum, r0, r1, rows, P<int32_t>(row_idx), P<int32_t>(elem_idx), P<int32_t>(pos), P<uint32_t>(pos_valid));
        auto out = std::make_shared<Batch>();
        out->num_rows = rows;
        for (int c : required) out->cols.push_back(take(t.ctx, *cur.batch->cols[(size_t)c], P<int32_t>(row_idx), rows, false));
        if (func == GEN_POS_EXPLODE) {
            auto pc = std::make_shared<Column>();
            pc->type = DType(T_INT32);
            pc->len = rows;
            pc->data = pos;
            if (pos_valid) {
                pc->validity = pos_valid;
                pc->null_count = -1;
            }
            out->cols.push_back(pc);
        }
        out->cols.push_back(take(t.ctx, *list->child, P<int32_t>(elem_idx), rows, outer));
        metrics.add("output_rows", rows);
        return out;
    }
}

// ------------------------------------------------------------------------------------------ ExpandExec
ExpandExec::ExpandExec(OperatorPtr input, const Schema& schema, std::vector<std::vector<ExprPtr>> projs) : projections(std::move(projs)) {
    name = "ExpandExec";
    out_schema = schema;
    const Schema& in = input->out_schema;
    AURON_CHECK(!projections.empty(), "ExpandExecNode without projections");
    for (auto& pr : projections) {
        AURON_CHECK(pr.size() == schema.fields.size(), "ExpandExec: a projection does not match the output schema");
        std::vector<ExprPtr> computed;
        std::vector<int> pl;
        for (size_t i = 0; i < pr.size(); i++) {
            const DType actual = infer_type(*pr[i], in);
            if (actual != schema.fields[i].type) {   // expand_exec.rs:166-168
                auto c = std::make_shared<Expr>();
                c->kind = E_TRY_CAST;
                c->type = schema.fields[i].type;
                c->children.push_back(pr[i]);
                pr[i] = c;
            }
            int idx = -1;
            if (is_plain_column(*pr[i], in, &idx)) pl.push_back(idx);
            else {
                pl.push_back(-1);
                computed.push_back(pr[i]);
            }
        }
        plain.push_back(pl);
        progs.push_back(computed.empty() ? VmProgram() : compile_projection(computed, in));
    }
    children.push_back(std::move(input));
}
std::string ExpandExec::describe() const {
    std::string o = "\"projections\":[";
    for (size_t i = 0; i < projections.size(); i++) o += (i ? "," : "") + exprs_json(projections[i]);
    return o + "]";
}
BatchPtr ExpandExec::next(Task& t) {
    if (!cur || next_proj >= projections.size()) {
        cur = children[0]->next(t);
        next_proj = 0;
        if (!cur) return nullptr;
    }
    OpTimer timer(metrics, "elapsed_ns");
    const size_t pi = next_proj++;
    auto out = std::make_shared<Batch>();
    out->num_rows = cur->num_rows;
    std::vector<ColumnPtr> computed;
    if (progs[pi].impl) computed = eval_projection(t.ctx, progs[pi], *cur, nullptr, cur->num_rows);
    size_t ci = 0;
    for (int idx : plain[pi]) out->cols.push_back(idx >= 0 ? cur->cols[(size_t)idx] : computed[ci++]);
    if (next_proj >= projections.size()) cur.reset();
    metrics.add("output_rows", out->num_rows);
    return out;
}

// ------------------------------------------------------------------------------------------ AggExec
static bool load_compatible(const DType& child, const DType& acc) {
    if (child == acc) return true;
    if (acc.id == T_INT64 && child.is_integer()) return true;
    if (acc.id == T_FLOAT64 && (child.is_integer() || child.is_float())) return true;
    if (acc.id == T_DECIMAL128 && child.id == T_DECIMAL128 && child.scale == acc.scale) return true;
    return false;
}

AggExec::AggExec(OperatorPtr input, std::vector<ExprPtr> ge, std::vector<std::string> gn, std::vector<AggExprSpec> ag)
    : group_exprs(std::move(ge)), group_names(std::move(gn)), aggs(std::move(ag)) {
    name = "AggExec";
    const Schema& in = input->out_schema;
    bool any_final = false, any_nonfinal = false;
    for (auto& a : aggs) {
        if (a.mode == MODE_FINAL) any_final = true;
        else any_nonfinal = true;
    }
    AURON_CHECK(!(any_final && any_nonfinal), "final aggregates may not be mixed with partial ones (agg_ctx.rs:111)");
    is_final = any_final;
    // accumulator layouts (acc_array_data_types of agg/sum.rs, count.rs, avg.rs:52, maxmin.rs, first.rs:50)
    input_acc_cols = 0;
    for (auto& a : aggs) {
        switch (a.fn) {
            case AGG_SUM: a.acc_types = {a.return_type}; break;
            case AGG_COUNT: a.acc_types = {DType(T_INT64)}; break;
            case AGG_AVG: a.acc_types = {a.return_type, DType(T_INT64)}; break;
            case AGG_MIN: case AGG_MAX: case AGG_FIRST: case AGG_FIRST_IGNORES_NULL: a.acc_types.clear(); break;
            default: fail("aggregate function " + std::to_string(a.fn) + " is not native on device (collect/bloom/UDAF are out of scope)");
        }
        if (a.mode != MODE_PARTIAL) input_acc_cols += (a.fn == AGG_FIRST) ? 2 : (a.acc_types.empty() ? 1 : (int)a.acc_types.size());
        AURON_CHECK(a.mode == MODE_PARTIAL || a.mode == MODE_PARTIAL_MERGE || a.mode == MODE_FINAL, "unknown aggregate mode");
        AURON_CHECK(a.mode != MODE_PARTIAL || a.fn == AGG_COUNT || !a.children.empty(), "aggregate function without an argument");   // COUNT() counts rows
    }
    // value types for MIN/MAX/FIRST: child type in partial mode, the trailing acc column type in merge modes
    int acc_pos = (int)in.fields.size() - input_acc_cols;
    AURON_CHECK(acc_pos >= 0, "aggregate input has fewer columns than accumulator arrays");
    for (auto& a : aggs) {
        bool value_typed = a.fn == AGG_MIN || a.fn == AGG_MAX || a.fn == AGG_FIRST || a.fn == AGG_FIRST_IGNORES_NULL;
        if (value_typed) {
            if (a.mode == MODE_PARTIAL) a.value_type = infer_type(*a.children[0], in);
            else {
                AURON_CHECK(acc_pos < (int)in.fields.size(), "aggregate input has fewer columns than accumulator arrays");
                a.value_type = in.fields[acc_pos].type;
            }
            a.acc_types = {a.value_type};
            if (a.fn == AGG_FIRST) a.acc_types.push_back(DType(T_BOOL));
        }
        if (a.mode != MODE_PARTIAL) acc_pos += (int)a.acc_types.size();
    }
    // lowered input expressions: group keys, then the args of every partial-mode aggregate
    for (auto& g : group_exprs) lowered.push_back(g);
    // GROUP BY cast(int column AS wider int): the widening is injective, so group on the source column (fast 64-bit key
    // path sign-extends it anyway) and emit the key in the wider type -- saves materialising the cast for every input row.
    if (group_exprs.size() == 1 && (group_exprs[0]->kind == E_CAST || group_exprs[0]->kind == E_TRY_CAST)) {
        int idx;
        const Expr& ce = *group_exprs[0];
        if (is_plain_column(*ce.children[0], in, &idx)) {
            const DType& from = in.fields[idx].type;
            if (from.is_integer() && ce.type.is_integer() && from.width() <= ce.type.width()) {
                lowered[0] = ce.children[0];
                widened_key_type = ce.type;
                has_widened_key = true;
            }
        }
    }
    for (auto& a : aggs) {
        if (a.mode != MODE_PARTIAL) continue;
        for (size_t k = 0; k < a.children.size(); k++) {
            ExprPtr e = a.children[k];
            if (k == 0 && (a.fn == AGG_SUM || a.fn == AGG_AVG)) {   // agg.rs:191-198 TryCast(child, return_type)
                DType ct = infer_type(*e, in);
                if (!load_compatible(ct, a.return_type)) {
                    auto c = std::make_shared<Expr>();
                    c->kind = E_TRY_CAST;
                    c->type = a.return_type;
                    c->children.push_back(e);
                    e = c;
                }
            }
            lowered.push_back(e);
        }
    }
    for (auto& e : lowered) {
        int idx = -1;
        if (is_plain_column(*e, in, &idx)) lowered_plain.push_back(idx);
        else {
            lowered_plain.push_back(-1);
            all_plain = false;
        }
    }
    if (!all_plain) lowered_prog = compile_projection(lowered, in);
    // output schema (agg_ctx.rs:127-150)
    for (size_t i = 0; i < group_exprs.size(); i++) {
        Field f;
        f.name = i < group_names.size() ? group_names[i] : "";
        f.type = infer_type(*group_exprs[i], in);
        out_schema.fields.push_back(f);
    }
    for (auto& a : aggs) {
        if (is_final) {
            Field f;
            f.name = a.name;
            f.type = (a.fn == AGG_COUNT) ? DType(T_INT64) : (a.fn == AGG_SUM || a.fn == AGG_AVG) ? a.return_type : a.value_type;
            out_schema.fields.push_back(f);
        } else {
            for (auto& at : a.acc_types) {
                Field f;
                f.name = "";
                f.type = at;
                out_schema.fields.push_back(f);
            }
        }
    }
    n_acc_cols = 0;
    for (auto& a : aggs) n_acc_cols += (int)a.acc_types.size();
    children.push_back(std::move(input));
}

static AccKind sum_kind(const DType& acc) {
    if (acc.id == T_DECIMAL128) return ACC_SUM_DEC;
    if (acc.id == T_FLOAT64 || acc.id == T_FLOAT32) return ACC_SUM_F64;
    return ACC_SUM_I64;
}

// build accumulator specs.  `merge_cols` != nullptr: every aggregate merges from these acc columns.
static std::vector<AccSpec> build_specs(const std::vector<AggExprSpec>& aggs, const std::vector<ColumnPtr>& partial_args,
                                        const std::vector<ColumnPtr>* merge_cols, bool force_merge) {
    std::vector<AccSpec> specs;
    size_t pa = 0, mc = 0;
    for (auto& a : aggs) {
        bool merge = force_merge || a.mode != MODE_PARTIAL;
        if (!merge) {
            size_t nargs = a.children.size();
            std::vector<ColumnPtr> args(partial_args.begin() + pa, partial_args.begin() + pa + nargs);
            pa += nargs;
            switch (a.fn) {
                case AGG_SUM: specs.push_back({sum_kind(a.acc_types[0]), args[0], {}, a.acc_types[0], nullptr}); break;
                case AGG_COUNT: {
                    AccSpec s{ACC_COUNT, args.empty() ? nullptr : args[0], {}, DType(T_INT64), nullptr};
                    for (size_t k = 1; k < args.size(); k++) s.extra.push_back(args[k]);
                    specs.push_back(s);
                    break;
                }
                case AGG_AVG:
                    specs.push_back({sum_kind(a.acc_types[0]), args[0], {}, a.acc_types[0], nullptr});
                    specs.push_back({ACC_COUNT, args[0], {}, DType(T_INT64), nullptr});
                    break;
                case AGG_MIN: specs.push_back({args[0]->type.is_varlen() ? ACC_MIN_STR : ACC_MIN, args[0], {}, a.value_type, nullptr}); break;
                case AGG_MAX: specs.push_back({args[0]->type.is_varlen() ? ACC_MAX_STR : ACC_MAX, args[0], {}, a.value_type, nullptr}); break;
                case AGG_FIRST: specs.push_back({ACC_FIRST, args[0], {}, a.value_type, nullptr}); break;
                case AGG_FIRST_IGNORES_NULL: specs.push_back({ACC_FIRST_IGNORES_NULL, args[0], {}, a.value_type, nullptr}); break;
            }
        } else {
            const std::vector<ColumnPtr>& m = *merge_cols;
            switch (a.fn) {
                case AGG_SUM: specs.push_back({sum_kind(a.acc_types[0]), m[mc], {}, a.acc_types[0], nullptr}); mc += 1; break;
                case AGG_COUNT: specs.push_back({ACC_ADD_I64, m[mc], {}, DType(T_INT64), nullptr}); mc += 1; break;
                case AGG_AVG:
                    specs.push_back({sum_kind(a.acc_types[0]), m[mc], {}, a.acc_types[0], nullptr});
                    specs.push_back({ACC_ADD_I64, m[mc + 1], {}, DType(T_INT64), nullptr});
                    mc += 2;
                    break;
                case AGG_MIN: specs.push_back({m[mc]->type.is_varlen() ? ACC_MIN_STR : ACC_MIN, m[mc], {}, a.value_type, nullptr}); mc += 1; break;
                case AGG_MAX: specs.push_back({m[mc]->type.is_varlen() ? ACC_MAX_STR : ACC_MAX, m[mc], {}, a.value_type, nullptr}); mc += 1; break;
                case AGG_FIRST: specs.push_back({ACC_FIRST, m[mc], {m[mc + 1]}, a.value_type, nullptr}); mc += 2; break;
                case AGG_FIRST_IGNORES_NULL: specs.push_back({ACC_FIRST_IGNORES_NULL, m[mc], {}, a.value_type, nullptr}); mc += 1; break;
            }
        }
    }
    return specs;
}

static BatchPtr run_agg(Task& t, const std::vector<ColumnPtr>& keys, const std::vector<AccSpec>& specs, const int32_t* sel, int64_t n,
                        const DType* key_out = nullptr, const uint32_t* selmask = nullptr, int64_t n_selected = -1) {
    auto out = std::make_shared<Batch>();
    if (keys.empty()) {
        auto accs = global_aggregate(t.ctx, specs, sel, n, selmask);
        out->num_rows = 1;
        out->cols = accs;
    } else {
        GroupedResult r = hash_aggregate(t.ctx, keys, specs, sel, n, key_out, selmask, n_selected);
        out->num_rows = r.num_groups;
        out->cols = r.keys->cols;
        for (auto& c : r.accs) out->cols.push_back(c);
    }
    return out;
}

BatchPtr AggExec::aggregate_chunk(Task& t, SelBatch& s) {
    const Batch& in = *s.batch;
    // plain column arguments: the kernels read the filter's bit mask directly; computed arguments need row indices
    const uint32_t* selmask = (all_plain && !s.sel) ? P<uint32_t>(s.mask) : nullptr;
    const int64_t n_selected = s.n;
    const int32_t* sel = selmask ? nullptr : ensure_sel(t, s);
    int64_t n = selmask ? in.num_rows : s.n;
    std::vector<ColumnPtr> lowered_cols;
    bool any_merge = false;
    for (auto& a : aggs) any_merge |= a.mode != MODE_PARTIAL;
    BatchPtr dense_holder;
    const Batch* src = &in;
    if (all_plain) {
        for (int idx : lowered_plain) lowered_cols.push_back(in.cols[idx]);
    } else {
        lowered_cols = eval_projection(t.ctx, lowered_prog, in, sel, n);
        if (sel && any_merge) {   // merge inputs must line up with the dense lowered columns
            dense_holder = take_batch(t.ctx, in, sel, n, false);
            src = dense_holder.get();
        }
        sel = nullptr;
    }
    std::vector<ColumnPtr> keys(lowered_cols.begin(), lowered_cols.begin() + group_exprs.size());
    std::vector<ColumnPtr> pargs(lowered_cols.begin() + group_exprs.size(), lowered_cols.end());
    std::vector<ColumnPtr> merge_cols;
    if (any_merge) {
        int start = (int)src->cols.size() - input_acc_cols;
        for (int i = start; i < (int)src->cols.size(); i++) merge_cols.push_back(src->cols[i]);
    }
    auto specs = build_specs(aggs, pargs, &merge_cols, false);
    return run_agg(t, keys, specs, sel, n, has_widened_key ? &widened_key_type : nullptr, selmask, n_selected);
}

BatchPtr AggExec::merge_partials(Task& t, const BatchPtr& all) {
    size_t g = group_exprs.size();
    std::vector<ColumnPtr> keys(all->cols.begin(), all->cols.begin() + g);
    std::vector<ColumnPtr> merge_cols(all->cols.begin() + g, all->cols.end());
    auto specs = build_specs(aggs, {}, &merge_cols, true);
    return run_agg(t, keys, specs, nullptr, all->num_rows);
}

BatchPtr AggExec::finalize(Task& t, const BatchPtr& merged) {
    if (!is_final) return merged;
    auto out = std::make_shared<Batch>();
    out->num_rows = merged->num_rows;
    size_t g = group_exprs.size(), pos = g;
    for (size_t i = 0; i < g; i++) out->cols.push_back(merged->cols[i]);
    for (auto& a : aggs) {
        switch (a.fn) {
            case AGG_AVG:
                out->cols.push_back(avg_finalize(t.ctx, *merged->cols[pos], *merged->cols[pos + 1], a.return_type));
                pos += 2;
                break;
            case AGG_FIRST:
                out->cols.push_back(merged->cols[pos]);
                pos += 2;
                break;
            default:
                out->cols.push_back(merged->cols[pos]);
                pos += 1;
        }
    }
    return out;
}

static int64_t batch_device_bytes(const Batch& b) {
    int64_t n = 0;
    for (auto& c : b.cols)
        for (const Buf* buf : {&c->validity, &c->data, &c->offsets})
            if (*buf) n += (int64_t)(*buf)->bytes;
    return n;
}

AggExec::~AggExec() {
    for (auto& pieces : spilled)
        for (auto& a : pieces)
            if (a.release) a.release(&a);
    if (mem_id) MemManager::of(mem_device).remove(mem_id);
}

// AggTable::spill (agg_table.rs:323-353): the in-memory table is emptied into `spill_buckets` hash buckets (bucket = pmod
// of the Spark murmur3 of the group keys, the same partitioner the shuffle uses) so that each bucket can later be merged on
// its own.  The next memory tier of a GPU node is pinned host DRAM, so the buckets are kept there as plain Arrow buffers:
// no serialization, no compression, D2H at PCIe rate.
void AggExec::spill(Task& t) {
    if (partials.empty()) return;
    OpTimer timer(metrics, "spill_ns");
    BatchPtr all = partials.size() == 1 ? partials[0] : merge_partials(t, concat_batches(t.ctx, partials));
    partials.clear();
    partial_rows = 0;
    if (all->num_rows == 0) return;
    if (spilled.empty()) {
        spilled.resize((size_t)spill_buckets);
        spill_schema.fields.clear();
        for (size_t i = 0; i < all->cols.size(); i++) {
            Field f;
            f.name = "c" + std::to_string(i);
            f.type = all->cols[i]->type;
            spill_schema.fields.push_back(f);
        }
    }
    std::vector<ColumnPtr> keys(all->cols.begin(), all->cols.begin() + group_exprs.size());
    Buf pids = murmur3_partition_ids(t.ctx, keys, all->num_rows, spill_buckets, 42);
    Buf rows, offs;
    partition_rows(t.ctx, P<int32_t>(pids), all->num_rows, spill_buckets, &rows, &offs);
    std::vector<int64_t> off((size_t)spill_buckets + 1, 0);
    to_host(t.ctx, off.data(), offs->ptr, off.size() * 8);
    BatchPtr sorted = take_batch(t.ctx, *all, P<int32_t>(rows), all->num_rows, false);
    int64_t bytes = 0;
    for (int b = 0; b < spill_buckets; b++) {
        int64_t n = off[(size_t)b + 1] - off[(size_t)b];
        if (n == 0) continue;
        BatchPtr piece = slice_batch(t.ctx, *sorted, off[(size_t)b], n);
        bytes += batch_device_bytes(*piece);
        ArrowArray a;
        memset(&a, 0, sizeof(a));
        export_batch(t.ctx, *piece, spill_schema, &a, (size_t)64 << 20);   // a pooled pinned block is >= 64 MB: only pieces that fill one
        spilled[(size_t)b].push_back(a);
    }
    metrics.add("mem_spill_count", 1);
    metrics.add("mem_spill_size", bytes);
}

// AggTable::output after a spill (agg_table.rs:145-304): every bucket is merged by itself and emitted as one batch
BatchPtr AggExec::next_spilled_bucket(Task& t) {
    while (out_bucket < spill_buckets) {
        auto& pieces = spilled[(size_t)out_bucket++];
        if (pieces.empty()) continue;
        std::vector<BatchPtr> parts;
        for (auto& a : pieces) {
            parts.push_back(import_batch(t.ctx, &a, spill_schema));
            if (a.release) a.release(&a);
        }
        pieces.clear();
        BatchPtr merged = merge_partials(t, parts.size() == 1 ? parts[0] : concat_batches(t.ctx, parts));
        BatchPtr out = finalize(t, merged);
        metrics.add("output_rows", out->num_rows);
        return out;
    }
    return nullptr;
}

// one input batch (with its pending selection) into the partial list
void AggExec::consume(Task& t, SelBatch& s) {
    if (s.n == 0 && !group_exprs.empty()) return;
    BatchPtr p = aggregate_chunk(t, s);
    partials.push_back(p);
    partial_rows += p->num_rows;
    // keep the partial list bounded: re-merge when it outgrows one chunk
    if (partials.size() > 1 && partial_rows > t.ctx.gpu_chunk_rows) {
        BatchPtr m = merge_partials(t, concat_batches(t.ctx, partials));
        partials.clear();
        partials.push_back(m);
        partial_rows = m->num_rows;
    }
    if (!group_exprs.empty()) {
        int64_t held = 0;
        for (auto& b : partials) held += batch_device_bytes(*b);
        if (spill_budget > 0) {   // an explicit budget for this operator (AURON_AGG_SPILL_BYTES)
            if (held > spill_budget) spill(t);
        } else {                  // the device-wide budget shared with every other spillable consumer (mem_manager.h)
            MemManager& mm = MemManager::of(t.ctx.device);
            if (!mem_id) {
                mem_id = mm.add("AggExec");
                mem_device = t.ctx.device;
            }
            if (mm.update(mem_id, held)) {
                spill(t);
                mm.update(mem_id, 0);
            }
        }
    }
}

// Can this aggregate, its optional FilterExec child and the scan below run as the fused pass?  Single integer group key that
// is a scan column (possibly under a widening cast), partial-mode SUM(int) / COUNT / MIN / MAX over scan columns, predicates
// that fold into per-column intervals; everything else keeps the operator-by-operator path.
void AggExec::setup_fusion() {
    fuse_checked = true;
    if (getenv("AURON_DISABLE_FUSED_SCAN_AGG")) return;
    if (group_exprs.size() != 1 || !all_plain || aggs.empty()) return;
    Operator* below = children[0].get();
    FilterExec* flt = dynamic_cast<FilterExec*>(below);
    if (flt) below = flt->children[0].get();
    FusedScanSource* src = dynamic_cast<FusedScanSource*>(below);
    if (!src) return;
    FusedAggSpec spec;
    if (flt && !predicate_intervals(flt->prog, &spec.pred_cols, &spec.pred_lo, &spec.pred_hi)) return;
    spec.key_col = lowered_plain[0];
    size_t pos = 1;
    for (auto& a : aggs) {
        if (a.mode != MODE_PARTIAL) return;
        FusedAggSpec::Acc acc;
        acc.col = a.children.empty() ? -1 : lowered_plain[pos];
        pos += a.children.size();
        switch (a.fn) {
            case AGG_SUM:
                if (a.acc_types[0].id != T_INT64) return;
                acc.kind = ACC_SUM_I64;
                acc.out_type = a.acc_types[0];
                break;
            case AGG_COUNT:
                if (a.children.size() > 1) return;
                acc.kind = ACC_COUNT;
                acc.out_type = DType(T_INT64);
                break;
            case AGG_MIN: case AGG_MAX:
                if (!(a.value_type.id == T_INT32 || a.value_type.id == T_DATE32 || a.value_type.id == T_INT64)) return;
                acc.kind = a.fn == AGG_MIN ? ACC_MIN : ACC_MAX;
                acc.out_type = a.value_type;
                break;
            default: return;
        }
        spec.accs.push_back(acc);
    }
    if (!src->can_fuse(spec)) return;
    fused_src = src;
    fused_filter = flt;
    fused_spec = spec;
}

BatchPtr AggExec::next(Task& t) {
    if (output_done) return spilled.empty() ? nullptr : next_spilled_bucket(t);
    bool saw_input = false;
    if (spill_budget == 0) {
        spill_budget = -1;   // no budget of its own: the device-wide MemManager decides (consume())
        if (const char* e = getenv("AURON_AGG_SPILL_BYTES")) spill_budget = atoll(e) > 0 ? atoll(e) : -1;
    }
    if (!fuse_checked) setup_fusion();
    while (!input_done && fused_src) {   // ParquetScan -> [Filter] -> this aggregate as one pass per batch (k_fused.cu)
        AURON_CHECK(t.is_running(), "task killed");
        OpTimer timer(metrics, "hashing_ns");
        BatchPtr fb;
        const int r = fused_src->next_fused(t, fused_spec, fused_state, &fb);
        if (r == FUSED_END) {
            input_done = true;
            if (fused_state.table) {
                if (direct_agg_out_of_range(t.ctx, *fused_state.table)) {
                    // the column statistics did not cover the key values (buggy writer): everything aggregated so far is void.
                    // Read the input again, operator by operator (that path detects lying statistics per chunk and falls back to its hash table).
                    AURON_CHECK(spilled.empty(), "parquet column statistics do not cover the values of the group key column");
                    fused_src->restart(t);
                    fused_src = nullptr;
                    fused_state = FusedAggState();
                    partials.clear();
                    partial_rows = 0;
                    input_done = false;
                    break;
                }
                unsigned long long counters[2] = {0, 0};   // rows that passed the predicates, tiles done by the TMA-staged kernel
                to_host(t.ctx, counters, fused_state.selected->ptr, 16);
                const unsigned long long sel_rows = counters[0];
                if (fused_filter) fused_filter->metrics.add("output_rows", (int64_t)sel_rows);
                metrics.add("fused_staged_tiles", (int64_t)counters[1]);
                metrics.add("fused_scan_rows", fused_state.rows);
                const DType key_type = has_widened_key ? widened_key_type : children[0]->out_schema.fields[(size_t)fused_spec.key_col].type;
                GroupedResult g = direct_agg_finish(t.ctx, *fused_state.table, key_type, fused_state.key_nullable);
                auto pb = std::make_shared<Batch>();
                pb->num_rows = g.num_groups;
                pb->cols = g.keys->cols;
                for (auto& c : g.accs) pb->cols.push_back(c);
                fused_state.table.reset();
                if (pb->num_rows) {
                    partials.push_back(pb);
                    partial_rows += pb->num_rows;
                }
            }
        } else if (r == FUSED_FALLBACK) {
            SelBatch s;
            if (fused_filter) s = fused_filter->apply(t, fb);
            else {
                s.batch = fb;
                s.n = fb->num_rows;
            }
            consume(t, s);
        }
    }
    while (!input_done) {
        AURON_CHECK(t.is_running(), "task killed");
        SelBatch s = children[0]->next_sel(t);
        if (!s.batch) {
            input_done = true;
            break;
        }
        saw_input = true;
        OpTimer timer(metrics, "hashing_ns");
        consume(t, s);
    }
    (void)saw_input;
    output_done = true;
    if (!spilled.empty()) {   // something was spilled: the rest follows it, then the buckets are merged one at a time
        spill(t);
        return next_spilled_bucket(t);
    }
    if (partials.empty()) {
        if (!group_exprs.empty()) return nullptr;
        // no grouping, no input: one row of empty accumulators (agg_exec.rs:280-323)
        SelBatch empty;
        auto eb = std::make_shared<Batch>();
        const Schema& in = children[0]->out_schema;
        for (auto& f : in.fields) eb->cols.push_back(f.type.is_varlen() ? make_column(t.ctx, f.type, 0, false) : make_column(t.ctx, f.type, 0, false));
        empty.batch = eb;
        empty.n = 0;
        partials.push_back(aggregate_chunk(t, empty));
    }
    BatchPtr merged = partials.size() == 1 ? partials[0] : merge_partials(t, concat_batches(t.ctx, partials));
    partials.clear();
    BatchPtr out = finalize(t, merged);
    metrics.add("output_rows", out->num_rows);
    return out;
}

// ------------------------------------------------------------------------------------------ HashJoinExec
HashJoinExec::HashJoinExec(OperatorPtr left, OperatorPtr right, std::vector<ExprPtr> lk, std::vector<ExprPtr> rk, int jt, int bs, const Schema& schema)
    : left_keys(std::move(lk)), right_keys(std::move(rk)), join_type(jt), build_side(bs) {
    name = "BroadcastJoin";   // BroadcastJoinExec::name() for shuffled-hash and broadcast joins alike (broadcast_join_exec.rs:243)
    out_schema = schema;
    if (out_schema.fields.empty()) {   // derive: [left cols..., right cols...] (full_join.rs:137-140)
        for (auto& f : left->out_schema.fields) out_schema.fields.push_back(f);
        if (jt == JOIN_EXISTENCE) {
            Field f;
            f.name = "exists";
            f.type = DType(T_BOOL);
            out_schema.fields.push_back(f);
        } else if (jt != JOIN_SEMI && jt != JOIN_ANTI) {
            for (auto& f : right->out_schema.fields) out_schema.fields.push_back(f);
        }
    }
    children.push_back(std::move(left));
    children.push_back(std::move(right));
}

static std::vector<ColumnPtr> eval_keys(Task& t, const std::vector<ExprPtr>& keys, const Schema& schema, const Batch& b) {
    std::vector<ColumnPtr> out;
    for (auto& k : keys) out.push_back(eval_to_column(t, k, schema, b));
    return out;
}

void HashJoinExec::build(Task& t) {
    std::vector<BatchPtr> bs;
    Operator& bc = build_child();
    while (BatchPtr b = bc.next(t)) {
        AURON_CHECK(t.is_running(), "task killed");
        if (b->num_rows) bs.push_back(b);
    }
    if (bs.empty()) {
        build_batch = std::make_shared<Batch>();
        for (auto& f : bc.out_schema.fields) build_batch->cols.push_back(make_column(t.ctx, f.type, 0, false));
    } else build_batch = concat_batches(t.ctx, bs);
    const auto& keys = build_side == SIDE_LEFT ? left_keys : right_keys;
    build_key_cols = eval_keys(t, keys, bc.out_schema, *build_batch);
    table = join_build(t.ctx, build_key_cols, build_batch->num_rows);
    matched_build = dalloc_zero(t.ctx, bitmap_alloc_bytes(build_batch->num_rows) + 4);
    built = true;
    metrics.add("build_rows", build_batch->num_rows);
}

static BatchPtr null_batch(Task& t, const Schema& s, int64_t n) {
    auto b = std::make_shared<Batch>();
    b->num_rows = n;
    for (auto& f : s.fields) {
        if (f.type.is_varlen()) {
            auto c = make_column(t.ctx, f.type, n, true);
            c->null_count = n;
            CUDA_OK(cudaMemsetAsync(c->offsets->ptr, 0, (size_t)(n + 1) * 4, t.ctx.stream));
            b->cols.push_back(c);
        } else b->cols.push_back(make_null_column(t.ctx, f.type, n));
    }
    return b;
}
static ColumnPtr bool_column_from_bits(Buf bits, int64_t n) {
    auto c = std::make_shared<Column>();
    c->type = DType(T_BOOL);
    c->len = n;
    c->data = bits;
    return c;
}

BatchPtr HashJoinExec::probe_chunk(Task& t, const BatchPtr& probe) {
    bool probe_is_left = build_side == SIDE_RIGHT;
    Operator& pc = probe_child();
    const auto& keys = probe_is_left ? left_keys : right_keys;
    auto pkeys = eval_keys(t, keys, pc.out_schema, *probe);
    int64_t n = probe->num_rows;
    bool probe_outer = (join_type == JOIN_FULL) || (join_type == JOIN_LEFT && probe_is_left) || (join_type == JOIN_RIGHT && !probe_is_left);
    bool semi_like = join_type == JOIN_SEMI || join_type == JOIN_ANTI || join_type == JOIN_EXISTENCE;
    if (semi_like) {
        Buf pm;
        join_probe(t.ctx, *table, pkeys, n, false, P<uint32_t>(matched_build), &pm);
        if (!probe_is_left) return nullptr;   // the build (left) side is emitted in finish()
        if (join_type == JOIN_EXISTENCE) {    // semi_join.rs:251-287: all probe rows + exists column
            auto out = std::make_shared<Batch>(*probe);
            out->cols.push_back(bool_column_from_bits(pm, n));
            return out;
        }
        Buf mask = pm;
        if (join_type == JOIN_ANTI) {
            if (null_aware_anti) {   // semi_join.rs:191-210: NOT IN drops everything when the build side has a NULL key
                if (join_table_has_null_key(*table)) return nullptr;
                Buf nn = not_bitmap(t.ctx, P<uint8_t>(pm), n);
                const uint8_t* kv = pkeys[0]->vbits();
                mask = kv ? and_bitmaps(t.ctx, P<uint8_t>(nn), kv, n) : nn;
            } else mask = not_bitmap(t.ctx, P<uint8_t>(pm), n);
        }
        int64_t cnt = 0;
        Buf idx = mask_to_indices(t.ctx, P<uint32_t>(mask), n, &cnt);
        if (cnt == 0) return nullptr;
        return take_batch(t.ctx, *probe, P<int32_t>(idx), cnt, false);
    }
    bool need_matched = (join_type == JOIN_FULL) || (join_type == JOIN_LEFT && !probe_is_left) || (join_type == JOIN_RIGHT && probe_is_left);
    JoinPairs pairs = join_probe(t.ctx, *table, pkeys, n, probe_outer, need_matched ? P<uint32_t>(matched_build) : nullptr, nullptr);
    if (pairs.count == 0) return nullptr;
    BatchPtr pcols = take_batch(t.ctx, *probe, P<int32_t>(pairs.probe_idx), pairs.count, false);
    BatchPtr bcols = take_batch(t.ctx, *build_batch, P<int32_t>(pairs.build_idx), pairs.count, probe_outer);
    auto out = std::make_shared<Batch>();
    out->num_rows = pairs.count;
    const BatchPtr& l = probe_is_left ? pcols : bcols;
    const BatchPtr& r = probe_is_left ? bcols : pcols;
    for (auto& c : l->cols) out->cols.push_back(c);
    for (auto& c : r->cols) out->cols.push_back(c);
    return out;
}

BatchPtr HashJoinExec::finish(Task& t) {
    bool probe_is_left = build_side == SIDE_RIGHT;
    int64_t nb = build_batch->num_rows;
    bool build_outer = (join_type == JOIN_FULL) || (join_type == JOIN_LEFT && !probe_is_left) || (join_type == JOIN_RIGHT && probe_is_left);
    bool semi_like = join_type == JOIN_SEMI || join_type == JOIN_ANTI || join_type == JOIN_EXISTENCE;
    if (semi_like) {
        if (probe_is_left || nb == 0) return nullptr;
        if (join_type == JOIN_EXISTENCE) {
            auto out = std::make_shared<Batch>(*build_batch);
            out->cols.push_back(bool_column_from_bits(matched_build, nb));
            return out;
        }
        Buf mask = join_type == JOIN_SEMI ? matched_build : not_bitmap(t.ctx, P<uint8_t>(matched_build), nb);
        int64_t cnt = 0;
        Buf idx = mask_to_indices(t.ctx, P<uint32_t>(mask), nb, &cnt);
        if (cnt == 0) return nullptr;
        return take_batch(t.ctx, *build_batch, P<int32_t>(idx), cnt, false);
    }
    if (!build_outer || nb == 0) return nullptr;
    // unmatched build rows (incl. NULL-key rows, join_hash_map.rs:103,331-338) with NULLs on the probe side
    Buf mask = not_bitmap(t.ctx, P<uint8_t>(matched_build), nb);
    int64_t cnt = 0;
    Buf idx = mask_to_indices(t.ctx, P<uint32_t>(mask), nb, &cnt);
    if (cnt == 0) return nullptr;
    BatchPtr bcols = take_batch(t.ctx, *build_batch, P<int32_t>(idx), cnt, false);
    BatchPtr pnull = null_batch(t, probe_child().out_schema, cnt);
    auto out = std::make_shared<Batch>();
    out->num_rows = cnt;
    const BatchPtr& l = probe_is_left ? pnull : bcols;
    const BatchPtr& r = probe_is_left ? bcols : pnull;
    for (auto& c : l->cols) out->cols.push_back(c);
    for (auto& c : r->cols) out->cols.push_back(c);
    return out;
}

SelBatch HashJoinExec::next_sel(Task& t) {
    SelBatch s;
    if (finished) return s;
    if (!built) build(t);
    const bool eligible = join_type == JOIN_INNER && table && join_table_unique_fast(*table) && !getenv("AURON_JOIN_NO_MASK");
    if (!eligible) {
        s.batch = next(t);
        s.n = s.batch ? s.batch->num_rows : 0;
        return s;
    }
    const bool probe_is_left = build_side == SIDE_RIGHT;
    while (!probe_done) {
        AURON_CHECK(t.is_running(), "task killed");
        BatchPtr p = probe_child().next(t);
        if (!p) {
            probe_done = true;
            break;
        }
        if (p->num_rows == 0) continue;
        OpTimer timer(metrics, "probed_side_compare_time");
        auto pkeys = eval_keys(t, probe_is_left ? left_keys : right_keys, probe_child().out_schema, *p);
        Buf idx, mask;
        const int64_t matched = join_probe_unique(t.ctx, *table, pkeys[0], p->num_rows, &idx, &mask);
        if (matched == 0) continue;
        BatchPtr bcols = take_batch(t.ctx, *build_batch, P<int32_t>(idx), p->num_rows, true);   // (-1 -> NULL: rows outside the mask)
        auto out = std::make_shared<Batch>();
        out->num_rows = p->num_rows;
        const BatchPtr& l = probe_is_left ? p : bcols;
        const BatchPtr& r = probe_is_left ? bcols : p;
        for (auto& c : l->cols) out->cols.push_back(c);
        for (auto& c : r->cols) out->cols.push_back(c);
        metrics.add("output_rows", matched);
        s.batch = out;
        s.n = matched;
        if (matched != p->num_rows) s.mask = mask;
        return s;
    }
    finished = true;
    return s;
}

BatchPtr HashJoinExec::next(Task& t) {
    if (finished) return nullptr;
    if (!built) build(t);
    while (!probe_done) {
        AURON_CHECK(t.is_running(), "task killed");
        BatchPtr p = probe_child().next(t);
        if (!p) {
            probe_done = true;
            break;
        }
        if (p->num_rows == 0) continue;
        BatchPtr out = probe_chunk(t, p);
        if (out && out->num_rows) {
            metrics.add("output_rows", out->num_rows);
            return out;
        }
    }
    finished = true;
    BatchPtr out = finish(t);
    if (out) metrics.add("output_rows", out->num_rows);
    return out;
}

// ------------------------------------------------------------------------------------------ WindowExec
WindowExec::WindowExec(OperatorPtr input, std::vector<ExprPtr> part, std::vector<ExprPtr> order, std::vector<WindowFuncSpec> fs, int64_t limit, bool out_cols)
    : partition_exprs(std::move(part)), order_exprs(std::move(order)), funcs(std::move(fs)), group_limit(limit), output_window_cols(out_cols) {
    name = "WindowExec";
    out_schema = input->out_schema;
    if (output_window_cols)
        for (auto& f : funcs) out_schema.fields.push_back(f.field);
    AURON_CHECK(group_limit < 0 || funcs.size() == 1, "WindowGroupLimit expects exactly one rank-like window function (window_exec.rs:341-344)");
    static const char* af[] = {"MIN", "MAX", "SUM", "AVG", "COUNT"};
    const Schema& is = input->out_schema;
    for (auto& f : funcs) {
        if (f.is_agg) {
            AURON_CHECK(f.func >= 0 && f.func <= 4, "window aggregate function #" + std::to_string(f.func) + " is not native in auron_b200 (MIN / MAX / SUM / AVG / COUNT are)");
            if (f.args.empty()) {   // COUNT(*)-like: every row counts
                AURON_CHECK(f.func == AGG_COUNT, std::string("window ") + af[f.func] + " without an argument");
                continue;
            }
            // the argument types of agg/{sum,avg,maxmin,count}.rs, checked when the plan is built
            const DType at = infer_type(*f.args[0], is);
            bool ok = true;
            if (f.func == AGG_SUM || f.func == AGG_AVG) ok = at.is_integer() || at.id == T_DATE32 || at.is_float() || at.id == T_DECIMAL128;
            else if (f.func == AGG_MIN || f.func == AGG_MAX) ok = at.is_intlike() || at.is_float() || at.id == T_DECIMAL128 || at.is_varlen() || at.id == T_BOOL;
            AURON_CHECK(ok, std::string("window ") + af[f.func] + " over " + at.str() + " is not supported");
            // SUM / AVG with a decimal result: TryCast(arg, return type) first, as AggExec does (agg.rs:191-198)
            if ((f.func == AGG_SUM || f.func == AGG_AVG) && f.field.type.id == T_DECIMAL128 && !load_compatible(at, f.field.type)) {
                auto c = std::make_shared<Expr>();
                c->kind = E_TRY_CAST;
                c->type = f.field.type;
                c->children.push_back(f.args[0]);
                f.args[0] = c;
            }
        } else {
            AURON_CHECK(f.func >= 0 && f.func <= 7, "window function #" + std::to_string(f.func) + " is not native in auron_b200");
            auto int_literal = [&](size_t i) { return f.args.size() > i && f.args[i]->kind == E_LITERAL && !f.args[i]->lit.is_null && f.args[i]->lit.type.width() > 0 && f.args[i]->lit.type.width() <= 8; };
            if (f.func == 3) AURON_CHECK(f.args.size() == 3 && int_literal(1), "LEAD expects input / literal integer offset / default children (lead_processor.rs:40-63)");
            if (f.func == 4 || f.func == 5) AURON_CHECK(f.args.size() == 2 && int_literal(1) && f.args[1]->lit.i > 0, "NTH_VALUE expects input / positive literal offset children (nth_value_processor.rs:36-66)");
            whole_partition = whole_partition || f.func == 3 || f.func == 6 || f.func == 7;   // window/mod.rs:115-120
        }
    }
    carries.resize(funcs.size());
    children.push_back(std::move(input));
}
std::string WindowExec::describe() const {
    std::string o = "\"partition_by\":[";
    for (size_t i = 0; i < partition_exprs.size(); i++) o += (i ? "," : "") + json_quote(expr_to_string(*partition_exprs[i]));
    o += "],\"order_by\":[";
    for (size_t i = 0; i < order_exprs.size(); i++) o += (i ? "," : "") + json_quote(expr_to_string(*order_exprs[i]));
    o += "],\"functions\":[";
    static const char* wf[] = {"ROW_NUMBER", "RANK", "DENSE_RANK", "LEAD", "NTH_VALUE", "NTH_VALUE_IGNORE_NULLS", "PERCENT_RANK", "CUME_DIST"};
    static const char* af[] = {"MIN", "MAX", "SUM", "AVG", "COUNT"};
    for (size_t i = 0; i < funcs.size(); i++) o += (i ? "," : "") + json_quote(std::string(funcs[i].is_agg ? af[funcs[i].func] : wf[funcs[i].func]) + " AS " + funcs[i].field.name);
    return o + "],\"group_limit\":" + std::to_string(group_limit) + ",\"output_window_cols\":" + (output_window_cols ? "true" : "false");
}
// rows [0, len) of a batch without a copy: the columns share the buffers (an Arrow array may have longer buffers than it uses)
static BatchPtr prefix_view(Task& t, const Batch& in, int64_t len) {
    auto out = std::make_shared<Batch>();
    out->num_rows = len;
    for (auto& c : in.cols) {
        auto v = std::make_shared<Column>(*c);
        v->len = len;
        if (c->null_count == c->len) v->null_count = len;
        else if (c->null_count != 0) v->null_count = -1;
        if (c->type.is_varlen()) {
            int32_t end = 0;
            to_host(t.ctx, &end, P<int32_t>(c->offsets) + len, 4);
            v->data_bytes = end;
        }
        out->cols.push_back(v);
    }
    return out;
}
BatchPtr WindowExec::take_staged(Task& t, const BatchPtr& extra) {
    std::vector<BatchPtr> parts;
    parts.swap(staged);
    staged_last.clear();
    if (extra) parts.push_back(extra);
    AURON_CHECK(!parts.empty(), "WindowExec: no rows held back");   // cut == 0 is only found against a held-back row
    if (parts.size() == 1) return parts[0];
    int64_t rows = 0;
    for (auto& b : parts) rows += b->num_rows;
    metrics.add("concat_rows", rows);
    return concat_batches(t.ctx, parts);
}
BatchPtr WindowExec::next(Task& t) {
    while (!done) {
        BatchPtr in = children[0]->next(t);
        AURON_CHECK(t.is_running(), "task killed");
        if (!in) {   // end of input: the rows held back form complete partitions
            done = true;
            if (staged.empty()) return nullptr;
            in = take_staged(t, nullptr);
        } else {
            if (in->num_rows == 0) continue;
            if (whole_partition) {
                // compute up to the last partition boundary and hold back the open partition (window_exec.rs:227-291); the held-back
                // batches are kept as they are and concatenated once, when their partition closes; without a partition spec all rows
                // are held back until the input ends
                if (partition_exprs.empty()) {
                    staged.push_back(in);
                    continue;
                }
                const int64_t n = in->num_rows;
                int64_t cut;
                std::vector<ColumnPtr> pk;
                {
                    OpTimer timer(metrics, "elapsed_ns");
                    for (auto& e : partition_exprs) pk.push_back(eval_to_column(t, e, children[0]->out_schema, *in));
                    // the last partition start in this batch; row 0 counts when it differs from the last held-back row
                    cut = window_last_boundary(t.ctx, pk, n, staged.empty() ? nullptr : &staged_last);
                }
                std::vector<ColumnPtr> last;
                for (auto& c : pk) last.push_back(slice_column(t.ctx, *c, n - 1, 1));
                if (cut < 0) {   // no partition closes here
                    staged.push_back(in);
                    staged_last = std::move(last);
                    continue;
                }
                // the held-back rows and rows [0, cut) form complete partitions; rows [cut, n) are the open one
                const BatchPtr batch = in;
                in = take_staged(t, cut > 0 ? prefix_view(t, *batch, cut) : nullptr);
                staged.push_back(cut > 0 ? slice_batch(t.ctx, *batch, cut, n - cut) : batch);
                staged_last = std::move(last);
            }
        }
        if (BatchPtr out = compute(t, in)) return out;
    }
    return nullptr;
}
BatchPtr WindowExec::compute(Task& t, const BatchPtr& in) {
    OpTimer timer(metrics, "elapsed_ns");
    const int64_t n = in->num_rows;
    const Schema& is = children[0]->out_schema;
    std::vector<ColumnPtr> pk, ok;
    for (auto& e : partition_exprs) pk.push_back(eval_to_column(t, e, is, *in));
    for (auto& e : order_exprs) ok.push_back(eval_to_column(t, e, is, *in));
    // row 0 continues the previous batch's partition (peer group) when its keys equal those of that batch's last row
    Buf pflags = window_boundaries(t.ctx, pk, n, nullptr, has_prev ? &prev_part : nullptr);
    Buf oflags = window_boundaries(t.ctx, ok, n, P<uint8_t>(pflags), has_prev ? &prev_order : nullptr);   // a new partition starts a new peer group
    std::vector<ColumnPtr> wcols;
    for (size_t i = 0; i < funcs.size(); i++) {
        const WindowFuncSpec& f = funcs[i];
        WinCarry* carry = &carries[i];
        if (!f.is_agg && f.func <= 2) {
            AURON_CHECK(f.field.type.id == T_INT32, "rank-like window functions return int32");
            wcols.push_back(window_rank_column(t.ctx, f.func, P<uint8_t>(pflags), P<uint8_t>(oflags), n, carry));
        } else if (!f.is_agg && (f.func == 6 || f.func == 7)) {
            AURON_CHECK(f.field.type.id == T_FLOAT64, "PERCENT_RANK / CUME_DIST return float64");
            wcols.push_back(window_dist_column(t.ctx, f.func, P<uint8_t>(pflags), P<uint8_t>(oflags), n));
        } else if (!f.is_agg && f.func == 3) {   // LEAD(input, offset, default)
            ColumnPtr vals = eval_to_column(t, f.args[0], is, *in);
            ColumnPtr dflt = (f.args[2]->kind == E_LITERAL && f.args[2]->lit.is_null) ? make_null_column(t.ctx, vals->type, n) : eval_to_column(t, f.args[2], is, *in);
            AURON_CHECK(dflt->type == vals->type, "LEAD: the default is " + dflt->type.str() + ", the input " + vals->type.str());
            wcols.push_back(window_lead_column(t.ctx, vals, dflt, f.args[1]->lit.i, P<uint8_t>(pflags), n));
        } else if (!f.is_agg) {                  // NTH_VALUE [IGNORE NULLS](input, n)
            ColumnPtr vals = eval_to_column(t, f.args[0], is, *in);
            wcols.push_back(window_nth_column(t.ctx, vals, f.args[1]->lit.i, f.func == 5, P<uint8_t>(pflags), n, carry));
        } else {
            ColumnPtr arg;
            if (f.args.empty()) arg = make_column(t.ctx, DType(T_INT8), n, false);   // COUNT(*)-like: every row counts
            else arg = eval_to_column(t, f.args[0], is, *in);
            wcols.push_back(window_agg_column(t.ctx, f.func, arg, f.field.type, P<uint8_t>(pflags), n, carry));
        }
    }
    prev_part.clear();
    prev_order.clear();
    for (auto& c : pk) prev_part.push_back(slice_column(t.ctx, *c, n - 1, 1));
    for (auto& c : ok) prev_order.push_back(slice_column(t.ctx, *c, n - 1, 1));
    has_prev = true;
    auto out = std::make_shared<Batch>();
    out->num_rows = n;
    out->cols = in->cols;
    if (output_window_cols)
        for (auto& c : wcols) out->cols.push_back(c);
    if (group_limit >= 0) {   // keep the rows whose rank is <= k (window_exec.rs:341-356); the rank carries across batches
        Buf mask = window_le_mask(t.ctx, wcols[0], (int32_t)std::min<int64_t>(group_limit, INT32_MAX));
        int64_t cnt = 0;
        Buf idx = mask_to_indices(t.ctx, P<uint32_t>(mask), n, &cnt);
        if (cnt == 0) return nullptr;
        if (cnt != n) out = take_batch(t.ctx, *out, P<int32_t>(idx), cnt, false);
    }
    metrics.add("output_rows", out->num_rows);
    return out;
}

// ------------------------------------------------------------------------------------------ SortMergeJoinExec
namespace {
struct BatchListExec : Operator {   // a fixed list of batches as an operator (one piece of one side)
    std::vector<BatchPtr> batches;
    size_t pos = 0;
    BatchListExec(const Schema& s, std::vector<BatchPtr> b) : batches(std::move(b)) {
        name = "SmjPiece";
        out_schema = s;
    }
    BatchPtr next(Task&) override { return pos < batches.size() ? batches[pos++] : nullptr; }
};
struct ForwardExec : Operator {     // forwards to an operator owned elsewhere
    Operator* target;
    explicit ForwardExec(Operator* o) : target(o) {
        name = o->name;
        out_schema = o->out_schema;
    }
    BatchPtr next(Task& t) override { return target->next(t); }
};
}  // namespace

SortMergeJoinExec::SortMergeJoinExec(OperatorPtr left, OperatorPtr right, std::vector<ExprPtr> lk, std::vector<ExprPtr> rk, std::vector<std::pair<bool, bool>> opts,
                                     int jt, const Schema& schema)
    : left_keys(std::move(lk)), right_keys(std::move(rk)), sort_opts(std::move(opts)), join_type(jt) {
    name = "SortMergeJoinExec";
    // output schema exactly as the hash join derives it: [left cols..., right cols...] (+ exists)
    HashJoinExec probe_schema(std::make_unique<BatchListExec>(left->out_schema, std::vector<BatchPtr>()),
                              std::make_unique<BatchListExec>(right->out_schema, std::vector<BatchPtr>()), left_keys, right_keys, jt, SIDE_RIGHT, schema);
    out_schema = probe_schema.out_schema;
    while (sort_opts.size() < left_keys.size()) sort_opts.emplace_back(true, true);   // SortOptions::default(): ascending, nulls first
    children.push_back(std::move(left));
    children.push_back(std::move(right));
}
std::string SortMergeJoinExec::describe() const {
    static const char* jt[] = {"INNER", "LEFT", "RIGHT", "FULL", "SEMI", "ANTI", "EXISTENCE"};
    return std::string("\"join_type\":\"") + (join_type >= 0 && join_type <= 6 ? jt[join_type] : "?") + "\",\"left_keys\":" + exprs_json(left_keys) +
           ",\"right_keys\":" + exprs_json(right_keys);
}
bool SortMergeJoinExec::pull(Task& t, int s) {
    if (side[s].done) return false;
    BatchPtr b = children[(size_t)s]->next(t);
    if (!b) {
        side[s].done = true;
        return false;
    }
    if (b->num_rows == 0) return true;
    side[s].buf = side[s].buf && side[s].buf->num_rows ? concat_batches(t.ctx, {side[s].buf, b}) : b;
    return true;
}
std::vector<Buf> SortMergeJoinExec::words_of(Task& t, int s, const BatchPtr& b) {
    const auto& keys = s == 0 ? left_keys : right_keys;
    std::vector<SortKeySpec> specs;
    for (size_t i = 0; i < keys.size(); i++) specs.push_back({eval_to_column(t, keys[i], children[(size_t)s]->out_schema, *b), sort_opts[i].first, sort_opts[i].second});
    std::vector<Buf> w;
    AURON_CHECK(sort_key_words(t.ctx, specs, b->num_rows, &w), "sort-merge join pieces need fixed-width keys");
    return w;
}
void SortMergeJoinExec::join_piece(Task& t, const BatchPtr& l, const BatchPtr& r) {
    // the driving side is probed (its order is the output order), the other side is built
    const int build = join_type == JOIN_RIGHT ? SIDE_LEFT : SIDE_RIGHT;
    std::vector<BatchPtr> lb, rb;
    if (l && l->num_rows) lb.push_back(l);
    if (r && r->num_rows) rb.push_back(r);
    HashJoinExec j(std::make_unique<BatchListExec>(children[0]->out_schema, lb), std::make_unique<BatchListExec>(children[1]->out_schema, rb), left_keys, right_keys, join_type,
                   build, Schema());
    while (BatchPtr b = j.next(t))
        if (b->num_rows) out_q.push_back(b);
    metrics.add("pieces", 1);
}
BatchPtr SortMergeJoinExec::next(Task& t) {
    if (!fallback_checked) {
        fallback_checked = true;
        bool varlen = false;
        for (auto& k : left_keys) varlen = varlen || infer_type(*k, children[0]->out_schema).is_varlen();
        for (auto& k : right_keys) varlen = varlen || infer_type(*k, children[1]->out_schema).is_varlen();
        if (varlen || getenv("AURON_SMJ_AS_HASH_JOIN")) {
            const int build = join_type == JOIN_RIGHT ? SIDE_LEFT : SIDE_RIGHT;
            whole.reset(new HashJoinExec(std::make_unique<ForwardExec>(children[0].get()), std::make_unique<ForwardExec>(children[1].get()), left_keys, right_keys, join_type,
                                         build, Schema()));
        }
    }
    if (whole) {
        BatchPtr b = whole->next(t);
        if (b) metrics.add("output_rows", b->num_rows);
        return b;
    }
    const int D = join_type == JOIN_RIGHT ? 1 : 0, O = 1 - D;
    for (;;) {
        if (out_pos < out_q.size()) {
            BatchPtr b = out_q[out_pos++];
            if (out_pos == out_q.size()) {
                out_q.clear();
                out_pos = 0;
            }
            metrics.add("output_rows", b->num_rows);
            return b;
        }
        if (finished) return nullptr;
        AURON_CHECK(t.is_running(), "task killed");
        // ---- 1. a piece of the driving side that ends at a key boundary
        if (!(side[D].buf && side[D].buf->num_rows) && !side[D].done) {
            pull(t, D);
            continue;
        }
        const bool d_empty = !(side[D].buf && side[D].buf->num_rows);
        BatchPtr dpiece, opiece;
        if (d_empty) {
            // the driving side is exhausted: what is left of the other side matches nothing; only FULL OUTER still emits it
            if (join_type != JOIN_FULL) {
                finished = true;
                continue;
            }
            if (!(side[O].buf && side[O].buf->num_rows) && !pull(t, O)) {
                if (side[O].done) finished = true;
                continue;
            }
            opiece = side[O].buf;
            side[O].buf.reset();
            if (opiece && opiece->num_rows) join_piece(t, D == 0 ? dpiece : opiece, D == 0 ? opiece : dpiece);
            continue;
        }
        std::vector<uint64_t> bound;   // key words (exclusive) below which every row of this piece lies; empty = unbounded
        {
            std::vector<Buf> w = words_of(t, D, side[D].buf);
            const int64_t n = side[D].buf->num_rows;
            std::vector<uint64_t> last(w.size());
            for (size_t i = 0; i < w.size(); i++) to_host(t.ctx, &last[i], P<uint64_t>(w[i]) + (n - 1), 8);
            if (side[D].done) {
                // last piece: everything buffered; the other side contributes the rows up to and including the last key
                dpiece = side[D].buf;
                side[D].buf.reset();
                bound = last;
                int i = (int)bound.size() - 1;
                while (i >= 0 && ++bound[(size_t)i] == 0) i--;   // tuple + 1 (lexicographic successor)
                if (i < 0) bound.clear();                        // the largest tuple there is: no upper bound
            } else {
                const int64_t cut = w.empty() ? 0 : lower_bound_sorted_words(t.ctx, w, n, last, 1)[0];
                if (cut == 0) {   // one key group so far: it may continue in the next batch
                    pull(t, D);
                    continue;
                }
                dpiece = slice_batch(t.ctx, *side[D].buf, 0, cut);
                side[D].buf = slice_batch(t.ctx, *side[D].buf, cut, n - cut);
                bound = last;
            }
        }
        // ---- 2. the rows of the other side below the bound
        for (;;) {
            const int64_t on = side[O].buf ? side[O].buf->num_rows : 0;
            if (on > 0 && !bound.empty()) {
                std::vector<Buf> w = words_of(t, O, side[O].buf);
                const int64_t ocut = lower_bound_sorted_words(t.ctx, w, on, bound, 1)[0];
                if (ocut < on || side[O].done) {   // a row at or above the bound is buffered: nothing below it can still arrive
                    opiece = ocut ? slice_batch(t.ctx, *side[O].buf, 0, ocut) : nullptr;
                    side[O].buf = ocut < on ? slice_batch(t.ctx, *side[O].buf, ocut, on - ocut) : nullptr;
                    break;
                }
            } else if (side[O].done) {
                opiece = side[O].buf;   // (unbounded: all of it)
                side[O].buf.reset();
                break;
            }
            pull(t, O);
        }
        join_piece(t, D == 0 ? dpiece : opiece, D == 0 ? opiece : dpiece);
    }
}

// ------------------------------------------------------------------------------------------ SortExec
SortExec::SortExec(OperatorPtr input, std::vector<SortExprSpec> k, int64_t lim, int64_t off) : keys(std::move(k)), limit(lim), offset(off) {
    name = "SortExec";
    out_schema = input->out_schema;
    children.push_back(std::move(input));
}
static void release_sort_runs(std::vector<SortExec::Run>& runs) {
    for (auto& r : runs)
        if (r.spilled && r.host.release) r.host.release(&r.host);
    runs.clear();
}
SortExec::~SortExec() {
    release_sort_runs(runs);
    if (mem_id) MemManager::of(mem_device).remove(mem_id);
}
BatchPtr SortExec::sort_batch(Task& t, const BatchPtr& in, int64_t keep_rows) {
    std::vector<SortKeySpec> specs;
    for (auto& k : keys) specs.push_back({eval_to_column(t, k.expr, out_schema, *in), k.asc, k.nulls_first});
    Buf perm = sort_indices(t.ctx, specs, in->num_rows);
    const int64_t n = keep_rows >= 0 ? std::min<int64_t>(keep_rows, in->num_rows) : in->num_rows;
    return take_batch(t.ctx, *in, P<int32_t>(perm), n, false);
}
static int64_t sort_batch_bytes(const Batch& b) {
    int64_t n = 0;
    for (auto& c : b.cols)
        for (const Buf* buf : {&c->validity, &c->data, &c->offsets})
            if (*buf) n += (int64_t)(*buf)->bytes;
    return n;
}
void SortExec::add_run(Task& t, const BatchPtr& sorted) {
    Run r;
    r.dev = sorted;
    r.rows = sorted->num_rows;
    r.bytes = sort_batch_bytes(*sorted);
    std::vector<SortKeySpec> specs;
    for (auto& k : keys) specs.push_back({eval_to_column(t, k.expr, out_schema, *sorted), k.asc, k.nulls_first});
    AURON_CHECK(sort_key_words(t.ctx, specs, sorted->num_rows, &r.words), "external sort over variable-length keys");
    memset(&r.host, 0, sizeof(r.host));
    runs.push_back(std::move(r));
    metrics.add("sorted_runs", 1);
}
// runs that do not fit the HBM budget move to pinned host memory, oldest first (sort_exec.rs:390-447: spill of the in-memory runs)
void SortExec::spill_if_needed(Task& t) {
    int64_t held = 0;
    for (auto& r : runs)
        if (!r.spilled) held += r.bytes;
    int64_t limit = spill_budget;
    if (spill_budget < 0) {   // the device-wide budget (mem_manager.h): when told to spill, give back down to half of what is held
        MemManager& mm = MemManager::of(t.ctx.device);
        if (!mem_id) {
            mem_id = mm.add("SortExec");
            mem_device = t.ctx.device;
        }
        limit = mm.update(mem_id, held) ? held / 2 : held;
    }
    for (auto& r : runs) {
        if (held <= limit) break;
        if (r.spilled) continue;
        OpTimer timer(metrics, "spill_ns");
        export_batch(t.ctx, *r.dev, out_schema, &r.host, (size_t)1 << 20);
        r.dev.reset();
        r.spilled = true;
        held -= r.bytes;
        metrics.add("mem_spill_count", 1);
        metrics.add("mem_spill_size", r.bytes);
    }
    if (mem_id) MemManager::of(t.ctx.device).update(mem_id, held);
}
// Splitters: every run contributes evenly spaced samples of its key words (each standing for rows / samples rows); the sorted
// sample is cut where the cumulated weight crosses a multiple of the target range size; every run is then cut at the splitters.
void SortExec::prepare_merge(Task& t) {
    merge_ready = true;
    int64_t total = 0;
    for (auto& r : runs) total += r.rows;
    const int64_t target = std::max<int64_t>(1, run_rows / 2);
    const int W = runs.empty() ? 0 : (int)runs[0].words.size();
    struct Sample {
        std::vector<uint64_t> w;
        double weight;
    };
    std::vector<Sample> samples;
    if (W > 0)
        for (auto& r : runs) {
            const int S = (int)std::min<int64_t>(r.rows, 1024);
            if (S <= 0) continue;
            std::vector<uint64_t> sw = sample_sorted_words(t.ctx, r.words, r.rows, S);
            for (int i = 0; i < S; i++) samples.push_back(Sample{std::vector<uint64_t>(sw.begin() + (size_t)i * W, sw.begin() + (size_t)(i + 1) * W), (double)r.rows / S});
        }
    std::sort(samples.begin(), samples.end(), [](const Sample& a, const Sample& b) { return a.w < b.w; });
    std::vector<uint64_t> splitters;   // [S][W], strictly increasing
    double acc = 0, next_cut = (double)target;
    const std::vector<uint64_t>* last = nullptr;
    for (auto& sm : samples) {
        acc += sm.weight;
        if (acc >= next_cut && acc < (double)total) {
            if (!last || *last < sm.w) {
                splitters.insert(splitters.end(), sm.w.begin(), sm.w.end());
                last = &sm.w;
            }
            while (next_cut <= acc) next_cut += (double)target;
        }
    }
    const int S = W ? (int)(splitters.size() / (size_t)W) : 0;
    n_ranges = (size_t)S + 1;
    for (auto& r : runs) {
        std::vector<int64_t> lb = S ? lower_bound_sorted_words(t.ctx, r.words, r.rows, splitters, S) : std::vector<int64_t>();
        r.cuts.assign(1, 0);
        for (int64_t v : lb) r.cuts.push_back(v);
        r.cuts.push_back(r.rows);
        r.words.clear();   // not needed any more
    }
    metrics.add("merge_ranges", (int64_t)n_ranges);
}
BatchPtr SortExec::window(const BatchPtr& b, Task& t) {
    // rows [offset, limit) of the whole sorted stream (sort_exec.rs:720-722,964)
    const int64_t first = emitted_seen, n = b->num_rows;
    emitted_seen += n;
    const int64_t lo = std::max<int64_t>(offset - first, 0), hi = limit >= 0 ? std::min<int64_t>(n, limit - first) : n;
    if (hi <= lo) return nullptr;
    if (lo == 0 && hi == n) return b;
    return slice_batch(t.ctx, *b, lo, hi - lo);
}
BatchPtr SortExec::next(Task& t) {
    if (done) return nullptr;
    if (run_rows == 0) {
        run_rows = t.ctx.gpu_chunk_rows;
        if (const char* e = getenv("AURON_SORT_RUN_ROWS")) run_rows = std::max<int64_t>(1, atoll(e));
        run_rows = std::min<int64_t>(run_rows, (int64_t)1 << 30);   // row ids inside a run are 32-bit
        spill_budget = -1;   // no budget of its own: the device-wide MemManager decides
        if (const char* e = getenv("AURON_SORT_SPILL_BYTES")) spill_budget = atoll(e) > 0 ? atoll(e) : -1;
    }
    bool varlen_key = false;
    for (auto& k : keys) varlen_key = varlen_key || infer_type(*k.expr, out_schema).is_varlen();
    // ---- run generation
    while (!input_done) {
        std::vector<BatchPtr> chunk;
        int64_t rows = 0;
        // (variable-length keys: one run holds everything -- their word count depends on the longest value, see sort_key_words)
        while (varlen_key || rows < run_rows) {
            AURON_CHECK(t.is_running(), "task killed");
            BatchPtr b = children[0]->next(t);
            if (!b) {
                input_done = true;
                break;
            }
            if (b->num_rows == 0) continue;
            // a batch larger than the run size is cut: runs stay within the 32-bit row ids of the sort kernels
            for (int64_t o = 0; o < b->num_rows; o += run_rows) {
                const int64_t m = std::min<int64_t>(run_rows, b->num_rows - o);
                chunk.push_back(m == b->num_rows ? b : slice_batch(t.ctx, *b, o, m));
                rows += m;
            }
        }
        if (chunk.empty()) break;
        // group the pieces into runs of at most run_rows rows
        size_t i = 0;
        while (i < chunk.size()) {
            std::vector<BatchPtr> grp;
            int64_t g = 0;
            while (i < chunk.size() && (grp.empty() || varlen_key || g + chunk[i]->num_rows <= run_rows)) {
                g += chunk[i]->num_rows;
                grp.push_back(chunk[i++]);
            }
            AURON_CHECK(g < (int64_t)INT32_MAX, "sort run too large (variable-length sort keys are sorted in one run)");
            OpTimer timer(metrics, "sort_ns");
            BatchPtr in = grp.size() == 1 ? grp[0] : concat_batches(t.ctx, grp);
            grp.clear();
            BatchPtr sorted = sort_batch(t, in, limit);   // only the first `limit` rows of a run can reach the output (sort_exec.rs:663)
            if (input_done && runs.empty() && i >= chunk.size()) {   // everything fitted one run: no merge
                done = true;
                BatchPtr out = window(sorted, t);
                if (out) metrics.add("output_rows", out->num_rows);
                return out;
            }
            add_run(t, sorted);
            spill_if_needed(t);
        }
    }
    if (runs.empty()) {
        done = true;
        return nullptr;
    }
    // ---- merge, one key range per call
    if (!merge_ready) prepare_merge(t);
    while (next_range < n_ranges) {
        const size_t r = next_range++;
        if (limit >= 0 && emitted_seen >= limit) break;
        OpTimer timer(metrics, "merge_ns");
        std::vector<BatchPtr> pieces;
        for (auto& run : runs) {
            const int64_t lo = run.cuts[r], n = run.cuts[r + 1] - lo;
            if (n <= 0) continue;
            pieces.push_back(run.spilled ? import_batch_slice(t.ctx, &run.host, out_schema, lo, n) : slice_batch(t.ctx, *run.dev, lo, n));
        }
        if (pieces.empty()) continue;
        BatchPtr in = pieces.size() == 1 ? pieces[0] : concat_batches(t.ctx, pieces);
        const bool single = pieces.size() == 1;
        pieces.clear();
        AURON_CHECK(in->num_rows < (int64_t)INT32_MAX, "a key range of the external sort exceeds 2^31 rows (one key value repeated that often?)");
        BatchPtr sorted = single ? in : sort_batch(t, in, -1);
        BatchPtr out = window(sorted, t);
        if (out) {
            metrics.add("output_rows", out->num_rows);
            return out;
        }
    }
    done = true;
    release_sort_runs(runs);
    return nullptr;
}

// ------------------------------------------------------------------------------------------ misc
LimitExec::LimitExec(OperatorPtr input, int64_t lim, int64_t off) : limit(lim), offset(off) {
    name = "LimitExec";
    out_schema = input->out_schema;
    children.push_back(std::move(input));
}
BatchPtr LimitExec::next(Task& t) {
    // rows [offset, limit) of the stream; stop pulling once satisfied (limit_exec.rs:132-180)
    while (seen < limit) {
        BatchPtr b = children[0]->next(t);
        if (!b) return nullptr;
        int64_t lo = std::max<int64_t>(offset - seen, 0), hi = std::min<int64_t>(b->num_rows, limit - seen);
        seen += b->num_rows;
        if (hi <= lo) continue;
        if (lo == 0 && hi == b->num_rows) return b;
        return slice_batch(t.ctx, *b, lo, hi - lo);
    }
    return nullptr;
}
RenameColumnsExec::RenameColumnsExec(OperatorPtr input, const std::vector<std::string>& names) {
    name = "RenameColumnsExec";
    out_schema = input->out_schema;
    for (size_t i = 0; i < names.size() && i < out_schema.fields.size(); i++) out_schema.fields[i].name = names[i];
    children.push_back(std::move(input));
}
PassThroughExec::PassThroughExec(OperatorPtr input, const std::string& nm) {
    name = nm;
    out_schema = input->out_schema;
    children.push_back(std::move(input));
}
UnionExec::UnionExec(std::vector<OperatorPtr> inputs, const Schema& schema) {
    name = "UnionExec";
    out_schema = schema;
    for (auto& i : inputs) children.push_back(std::move(i));
}
BatchPtr UnionExec::next(Task& t) {
    while (cur < children.size()) {
        BatchPtr b = children[cur]->next(t);
        if (b) return b;
        cur++;
    }
    return nullptr;
}

}  // namespace auron
