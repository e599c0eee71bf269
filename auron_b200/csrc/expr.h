// expr.h -- physical expression IR (mirror of auron.proto PhysicalExprNode :59-126 as resolved by
// PhysicalPlanner::try_parse_physical_expr, auron-planner/src/planner.rs:844-1053) and the compiler
// to the fused expression VM (k_expr.cu).
#pragma once
#include <map>

#include "common.h"

namespace auron {

struct Literal {
    DType type;
    bool is_null = true;
    int64_t i = 0;       // ints, dates, timestamps, bool
    double d = 0;        // floats
    uint64_t lo = 0;     // decimal128
    int64_t hi = 0;
    std::string s;       // utf8 / binary
};

enum ExprKind {
    E_COLUMN,      // name (resolved by name, planner.rs:855) or index (BoundReference)
    E_LITERAL,
    E_BINARY,      // op = proto string ("Plus", "Eq", "And", ... auron-planner/src/lib.rs:70-101)
    E_NOT,
    E_IS_NULL,
    E_IS_NOT_NULL,
    E_NEGATIVE,
    E_CASE,        // children: [expr?] (when, then)* [else?]; has_case_expr / has_else
    E_CAST,        // type = target
    E_TRY_CAST,
    E_IN_LIST,     // children[0] = expr, rest = list; negated
    E_SCALAR_FN,   // name = function name ("Spark_Year", "Substr", ...); type = return type
    E_LIKE,        // children: expr, pattern(literal); negated, case_insensitive
    E_STARTS_WITH, // children[0]; lit.s = prefix
    E_ENDS_WITH,
    E_CONTAINS,
    E_SC_AND,
    E_SC_OR,
    E_ROW_NUM,     // RowNumExprNode: int64 position of the row among the rows the projection emitted (row_num.rs)
};

struct HostArray;   // engine.h
struct Expr;
using ExprPtr = std::shared_ptr<Expr>;
struct Expr {
    ExprKind kind = E_LITERAL;
    std::vector<ExprPtr> children;
    std::string name;   // column / function name
    int index = -1;     // bound column index (-1 => resolve by name)
    std::string op;     // binary operator
    Literal lit;
    DType type;         // cast target / function return type
    std::shared_ptr<const HostArray> list_lit;   // E_LITERAL of a list type: the elements of the one list row (lit.is_null: NULL list)
    bool negated = false, case_insensitive = false, has_case_expr = false, has_else = false;
};

ExprPtr col(const std::string& name);
ExprPtr col_idx(int index);
ExprPtr lit_i64(int64_t v);
ExprPtr lit_null(const DType& t);

DType infer_type(const Expr& e, const Schema& input);
// the Spark string constructors (concat, concat_ws, repeat, space) and digests (md5, sha2) the projection compiler builds
bool makes_string_fn(const std::string& name);
// true when the expression is a bare column reference; *idx receives the resolved index
bool is_plain_column(const Expr& e, const Schema& input, int* idx);
// list values (list columns, list literals, Spark_StringSplit, Spark_MakeArray) are computed outside the VM, only as a whole
// projection expression or a generator's child (operators.cc ListExpr); the compilers reject them anywhere inside a program
bool is_list_fn(const std::string& name);
// keys evaluated only when the plan runs (sort, join, window, shuffle): rejected when the plan is built if a list value is among them
void reject_list_exprs(const std::vector<ExprPtr>& exprs, const Schema& input, const char* where);

// ---- compiled program -------------------------------------------------------------------
struct VmProgramImpl;
struct VmProgram {
    std::shared_ptr<VmProgramImpl> impl;
    std::vector<DType> out_types;   // one per output expression (empty for predicate programs)
    bool is_predicate = false;
};
// outputs = projection expressions; RowNum is accepted only with `row_num` (a ProjectExec, which passes its row count to
// eval_projection)
VmProgram compile_projection(const std::vector<ExprPtr>& exprs, const Schema& input, bool row_num = false);
// conjunction of predicates; NULL -> false (cached_exprs_evaluator.rs:514-519)
VmProgram compile_predicate(const std::vector<ExprPtr>& conjuncts, const Schema& input);

// conjunction folded into one closed interval per column (ordering comparisons against literals on non-decimal fixed-width
// columns): the columns (schema indices) and their bounds in the int64 domain; false when the predicate has another shape
bool predicate_intervals(const VmProgram& p, std::vector<int>* cols, std::vector<int64_t>* lo, std::vector<int64_t>* hi);

// evaluate over rows sel[0..n_out) (sel == nullptr: rows 0..n_out); RowNum gives row_base + the row's output position
std::vector<ColumnPtr> eval_projection(Ctx& ctx, const VmProgram& p, const Batch& in, const int32_t* sel, int64_t n_out, int64_t row_base = 0);
// returns selection bitmap (whole 32-bit words) over the n_rows input rows
Buf eval_predicate(Ctx& ctx, const VmProgram& p, const Batch& in, int64_t n_rows);

}  // namespace auron
