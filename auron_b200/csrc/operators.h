// operators.h -- operator classes (mirror of datafusion-ext-plans/src/*_exec.rs)
#pragma once
#include "arrow_bridge.h"
#include "engine.h"

namespace auron {

// proto enums (auron.proto)
enum AggFn { AGG_MIN = 0, AGG_MAX = 1, AGG_SUM = 2, AGG_AVG = 3, AGG_COUNT = 4, AGG_FIRST = 7, AGG_FIRST_IGNORES_NULL = 8 };
enum AggModeE { MODE_PARTIAL = 0, MODE_PARTIAL_MERGE = 1, MODE_FINAL = 2 };
enum JoinTypeE { JOIN_INNER = 0, JOIN_LEFT = 1, JOIN_RIGHT = 2, JOIN_FULL = 3, JOIN_SEMI = 4, JOIN_ANTI = 5, JOIN_EXISTENCE = 6 };
enum JoinSideE { SIDE_LEFT = 0, SIDE_RIGHT = 1 };

// ffi_reader_exec.rs: batches exported by the JVM (or HBM-resident batches registered under the id)
struct FFIReaderExec : Operator {
    std::string resource_id;
    bool is_device = false, done = false;
    std::vector<BatchPtr> dev_batches;
    size_t dev_pos = 0;
    FFIReaderExec(const Schema& schema, const std::string& id);
    std::string describe() const override;
    BatchPtr next(Task& t) override;
};

// ---- fused ParquetScan -> Filter -> HashAggregate (k_fused.cu): the handshake between AggExec and a scan that can run the
// three operators as one pass over the encoded pages.  The operator tree keeps its shape (metrics are reported per plan node,
// metrics.rs:22-50); AggExec pulls `next_fused` instead of `next_sel` when its own expressions, its FilterExec child's
// predicates and the scan's column types allow it.
struct FusedAggSpec {
    std::vector<int> pred_cols;              // scan output columns under a closed-interval test (NULL never passes)
    std::vector<int64_t> pred_lo, pred_hi;
    int key_col = -1;                        // scan output column of the single group key
    struct Acc {
        int kind;                            // AccKind: ACC_SUM_I64 / ACC_COUNT / ACC_MIN / ACC_MAX
        int col;                             // scan output column of the argument, -1 = COUNT(*)
        DType out_type;                      // accumulator column type
    };
    std::vector<Acc> accs;
};
struct FusedAggState {
    std::shared_ptr<DirectAgg> table;        // persistent direct-address table, widened batch by batch
    Buf selected;                            // device u64: rows that passed the predicates
    bool has_range = false, key_nullable = false;
    long long kmin = 0, kmax = -1;
    int64_t rows = 0, batches = 0;
};
enum { FUSED_END = 0, FUSED_DONE = 1, FUSED_FALLBACK = 2 };
struct FusedScanSource {
    virtual ~FusedScanSource() = default;
    virtual bool can_fuse(const FusedAggSpec& spec) const = 0;
    // FUSED_DONE: the next batch went through the fused kernels into `st`; FUSED_FALLBACK: it could not, *fallback holds it as
    // a regular batch; FUSED_END: no more input (all kernels of earlier batches have completed)
    virtual int next_fused(Task& t, const FusedAggSpec& spec, FusedAggState& st, BatchPtr* fallback) = 0;
    // rewind to the first row (after FUSED_END): the fused pass met keys outside the range the file statistics promised, its
    // result is void and the caller reads the input again through the regular path
    virtual void restart(Task& t) = 0;
};

// filter_exec.rs:128-224
struct FilterExec : Operator {
    std::vector<ExprPtr> predicates;
    VmProgram prog;
    FilterExec(OperatorPtr input, std::vector<ExprPtr> preds);
    std::string describe() const override;
    BatchPtr next(Task& t) override;
    SelBatch next_sel(Task& t) override;
    SelBatch apply(Task& t, const BatchPtr& b);   // the predicates over one batch
};

// A list-valued expression, computed outside the expression VM: a list column, a list literal, or Spark_StringSplit /
// Spark_MakeArray over flat arguments the VM computes.  Valid only as a whole projection expression or a generator's child.
struct ListExpr {
    enum Kind { COLUMN, LITERAL, SPLIT, MAKE_ARRAY } kind = COLUMN;
    DType type;                                  // the declared list type (its element field names the exported child)
    int col = -1;                                // COLUMN: input column
    std::vector<int> arg_slots;                  // SPLIT: the string, MAKE_ARRAY: the elements, as outputs of the caller's VM program
    std::string pattern;                         // SPLIT
    std::shared_ptr<const HostArray> lit;        // LITERAL: its elements (HostArray::list_is_null: the NULL list)
    ColumnPtr lit_dev;                           // LITERAL: the elements uploaded once
    std::string text;                            // the expression, for explain
};
// `e` as a ListExpr (its flat arguments appended to *args); false when `e` is not list-valued.  Rejects, naming the function,
// a list expression this engine does not compute.
bool plan_list_expr(const ExprPtr& e, const Schema& in, const DType& declared, ListExpr* out, std::vector<ExprPtr>* args);
// the list column of the n rows sel[0..n) (sel == nullptr: 0..n) of `b`; `computed` holds the program outputs over those rows
ColumnPtr eval_list_expr(Task& t, ListExpr& le, const Batch& b, const int32_t* sel, int64_t n, const std::vector<ColumnPtr>& computed);

// project_exec.rs:135-232 (fuses with a FilterExec child through next_sel)
struct ProjectExec : Operator {
    std::vector<ExprPtr> exprs;
    std::vector<int> plain_col;       // >= 0: bare column index, -1: computed
    std::vector<int> prog_slot;       // index into the VM program outputs for computed exprs
    std::vector<int> list_slot;       // >= 0: index into `lists` for list-valued exprs
    std::vector<ListExpr> lists;
    VmProgram prog;
    bool has_prog = false;
    int64_t rows_out = 0;             // rows emitted so far: the base of RowNum
    ProjectExec(OperatorPtr input, std::vector<ExprPtr> exprs, std::vector<std::string> names, std::vector<DType> types);
    std::string describe() const override;
    BatchPtr next(Task& t) override;
};

struct AggExprSpec {
    int fn = AGG_SUM;
    int mode = MODE_PARTIAL;
    std::vector<ExprPtr> children;
    DType return_type;
    std::string name;
    // derived
    std::vector<DType> acc_types;
    DType value_type;   // type of the aggregated values (MIN/MAX/FIRST)
};

// agg_exec.rs:141-323 + agg/*.rs
struct AggExec : Operator {
    std::vector<ExprPtr> group_exprs;
    std::vector<std::string> group_names;
    std::vector<AggExprSpec> aggs;
    bool is_final = false;
    bool input_done = false, output_done = false;
    std::vector<BatchPtr> partials;   // [group cols..., acc cols...]
    int64_t partial_rows = 0;
    // lowered input expressions (group keys + partial-mode agg args), evaluated through the VM when not plain
    std::vector<ExprPtr> lowered;
    std::vector<int> lowered_plain;
    bool all_plain = true;
    VmProgram lowered_prog;
    int n_acc_cols = 0, input_acc_cols = 0;
    bool has_widened_key = false;   // single GROUP BY cast(int col AS wider int): grouped on the source column
    DType widened_key_type;
    // memory-bounded table (agg_table.rs:99-135,323-353,474-721): when the partial results held in HBM outgrow the budget
    // they are split into hash buckets and moved to pinned host memory; the output then merges bucket by bucket
    int64_t spill_budget = 0;         // bytes of partials allowed to stay in HBM (0 = not yet sized, -1 = the device-wide MemManager decides)
    int mem_id = 0, mem_device = 0;   // consumer id at the MemManager of that device
    int spill_buckets = 64;
    std::vector<std::vector<ArrowArray>> spilled;   // [bucket] -> host-resident pieces ([group cols..., acc cols...])
    Schema spill_schema;
    int out_bucket = 0;
    // fused scan -> filter -> aggregate (see FusedScanSource)
    bool fuse_checked = false;
    FusedScanSource* fused_src = nullptr;
    FilterExec* fused_filter = nullptr;
    FusedAggSpec fused_spec;
    FusedAggState fused_state;
    AggExec(OperatorPtr input, std::vector<ExprPtr> group_exprs, std::vector<std::string> group_names, std::vector<AggExprSpec> aggs);
    ~AggExec() override;
    std::string describe() const override;
    BatchPtr next(Task& t) override;

   private:
    void spill(Task& t);
    void setup_fusion();
    void consume(Task& t, SelBatch& s);
    BatchPtr next_spilled_bucket(Task& t);
    BatchPtr aggregate_chunk(Task& t, SelBatch& s);
    BatchPtr merge_partials(Task& t, const BatchPtr& all);
    BatchPtr finalize(Task& t, const BatchPtr& merged);
};

// broadcast_join_exec.rs / sort_merge_join_exec.rs (hash build + probe for every join flavour)
struct HashJoinExec : Operator {
    std::vector<ExprPtr> left_keys, right_keys;
    int join_type = JOIN_INNER;
    int build_side = SIDE_RIGHT;
    bool null_aware_anti = false;
    std::string cache_id;
    // state
    bool built = false, probe_done = false, finished = false;
    BatchPtr build_batch;
    std::vector<ColumnPtr> build_key_cols;
    std::shared_ptr<JoinTable> table;
    Buf matched_build;
    HashJoinExec(OperatorPtr left, OperatorPtr right, std::vector<ExprPtr> lk, std::vector<ExprPtr> rk, int join_type, int build_side, const Schema& schema);
    std::string describe() const override;
    BatchPtr next(Task& t) override;
    // INNER join against a build side without duplicate keys (a dimension table on its primary key): the probe batch passes through
    // with a match mask and the build columns gathered beside it -- the probe columns are never copied (joins/bhj/full_join.rs:148-367
    // emits the same rows; consumers that skip rows themselves, the aggregate and the projection, take the mask as it is)
    SelBatch next_sel(Task& t) override;

   private:
    void build(Task& t);
    BatchPtr probe_chunk(Task& t, const BatchPtr& probe);
    BatchPtr finish(Task& t);
    Operator& build_child() { return *children[build_side == SIDE_LEFT ? 0 : 1]; }
    Operator& probe_child() { return *children[build_side == SIDE_LEFT ? 1 : 0]; }
};

// window_exec.rs:162-345 + window/processors/*.rs.  The input arrives sorted by (partition spec, order spec); every window function is a
// segmented scan (+ one scatter / gather for the functions that look at the whole partition) over one input batch (k_window.cu).
// Built: ROW_NUMBER, RANK, DENSE_RANK, PERCENT_RANK, CUME_DIST, LEAD, NTH_VALUE [IGNORE NULLS], running SUM / COUNT / MIN / MAX / AVG
// (SUM / AVG over integers, dates, floats and decimals; MIN / MAX also over strings, binary, booleans, date64 and timestamps),
// WindowGroupLimit (keep the rows with rank <= k) and output_window_cols = false.
// Batches stream through (window_exec.rs:224-304): the running functions carry their state at the last row into the next batch.
// When a function needs the whole partition (PERCENT_RANK, CUME_DIST, LEAD), the open partition at the end of a batch is held back
// and concatenated once with the rows that close it; without a partition spec that holds back the whole input.
struct WindowFuncSpec {
    bool is_agg = false;
    int func = 0;                 // WindowFunction (auron.proto:128-137) or AggFunction (MIN 0, MAX 1, SUM 2, AVG 3, COUNT 4)
    std::vector<ExprPtr> args;
    Field field;
};
struct WindowExec : Operator {
    std::vector<ExprPtr> partition_exprs, order_exprs;
    std::vector<WindowFuncSpec> funcs;
    int64_t group_limit = -1;
    bool output_window_cols = true, done = false;
    bool whole_partition = false;                // some function needs the whole partition
    std::vector<WinCarry> carries;               // per function
    bool has_prev = false;                       // a batch has been computed: prev_* hold the keys of its last row
    std::vector<ColumnPtr> prev_part, prev_order;
    std::vector<BatchPtr> staged;                // rows held back (whole_partition): the open partition, or all rows without a partition spec
    std::vector<ColumnPtr> staged_last;          // partition keys of the last held-back row (one row each)
    WindowExec(OperatorPtr input, std::vector<ExprPtr> part, std::vector<ExprPtr> order, std::vector<WindowFuncSpec> fs, int64_t limit, bool out_cols);
    std::string describe() const override;
    BatchPtr next(Task& t) override;

   private:
    BatchPtr compute(Task& t, const BatchPtr& in);   // the window columns of the next rows; nullptr when the group limit keeps none
    BatchPtr take_staged(Task& t, const BatchPtr& extra);   // the held-back rows (+ extra) as one batch, concatenated once
};

// sort_merge_join_exec.rs:135-205,294-372 + joins/smj/*.rs.  Both inputs arrive sorted on the join keys.  The reference advances two
// row cursors; here the two streams are cut into KEY-DISJOINT pieces (a piece ends where the key of the driving side changes, the
// other side contributes exactly the rows below that key) and every piece is joined with the hash kernels.  Memory is bounded
// by the piece (one input chunk per side plus the key group that straddles its end), both sides are streamed, and the output
// keeps the order of the driving side (left; right for RIGHT OUTER), which is what Spark assumes after a SortMergeJoin.
struct SortMergeJoinExec : Operator {
    std::vector<ExprPtr> left_keys, right_keys;
    std::vector<std::pair<bool, bool>> sort_opts;   // (asc, nulls_first) per key
    int join_type = JOIN_INNER;
    struct Side {
        BatchPtr buf;
        bool done = false;
    };
    Side side[2];   // 0 = left, 1 = right
    std::vector<BatchPtr> out_q;
    size_t out_pos = 0;
    bool finished = false, fallback_checked = false;
    std::unique_ptr<Operator> whole;   // variable-length keys: one hash join over the whole inputs (no key words to cut by)
    SortMergeJoinExec(OperatorPtr left, OperatorPtr right, std::vector<ExprPtr> lk, std::vector<ExprPtr> rk, std::vector<std::pair<bool, bool>> opts,
                      int join_type, const Schema& schema);
    std::string describe() const override;
    BatchPtr next(Task& t) override;

   private:
    bool pull(Task& t, int s);
    std::vector<Buf> words_of(Task& t, int s, const BatchPtr& b);
    void join_piece(Task& t, const BatchPtr& l, const BatchPtr& r);
};

struct SortExprSpec {
    ExprPtr expr;
    bool asc = true, nulls_first = true;
};
SortExprSpec decode_sort_expr(const uint8_t* b, size_t n);   // PhysicalExprNode{sort} (planner.cc)
// sort_exec.rs:197-290,637-768
struct SortExec : Operator {
    std::vector<SortExprSpec> keys;
    int64_t limit = -1, offset = 0;
    bool done = false;
    // ExternalSorter (sort_exec.rs:390-447,637-768,913-1061): the input is sorted in runs of at most `run_rows` rows; runs beyond
    // the HBM budget are spilled to pinned host memory; the output merges the runs key range by key range
    struct Run {
        BatchPtr dev;                 // sorted rows in HBM (null once spilled)
        ArrowArray host;              // pinned host copy (spilled runs)
        bool spilled = false;
        std::vector<Buf> words;       // normalised key words of the sorted rows (stay in HBM: 8..24 B per row)
        int64_t rows = 0, bytes = 0;
        std::vector<int64_t> cuts;    // [ranges + 1] row positions of the range boundaries
    };
    std::vector<Run> runs;
    bool input_done = false, merge_ready = false;
    int64_t run_rows = 0, spill_budget = 0, emitted_seen = 0;
    int mem_id = 0, mem_device = 0;   // consumer id at the MemManager (mem_manager.h)
    size_t next_range = 0, n_ranges = 0;
    SortExec(OperatorPtr input, std::vector<SortExprSpec> keys, int64_t limit, int64_t offset);
    ~SortExec() override;
    std::string describe() const override;
    BatchPtr next(Task& t) override;

   private:
    BatchPtr sort_batch(Task& t, const BatchPtr& in, int64_t keep_rows);   // rows of `in` in key order (first keep_rows of them; < 0 = all)
    void add_run(Task& t, const BatchPtr& sorted);
    void spill_if_needed(Task& t);
    void prepare_merge(Task& t);
    BatchPtr window(const BatchPtr& b, Task& t);   // rows of an output batch that fall into [offset, limit)
};

// limit_exec.rs:132-180
struct LimitExec : Operator {
    int64_t limit, offset, seen = 0, emitted = 0;
    LimitExec(OperatorPtr input, int64_t limit, int64_t offset);
    std::string describe() const override;
    BatchPtr next(Task& t) override;
};

struct RenameColumnsExec : Operator {
    RenameColumnsExec(OperatorPtr input, const std::vector<std::string>& names);
    BatchPtr next(Task& t) override { return children[0]->next(t); }
};
struct EmptyPartitionsExec : Operator {
    explicit EmptyPartitionsExec(const Schema& s) { name = "EmptyPartitionsExec"; out_schema = s; }
    BatchPtr next(Task&) override { return nullptr; }
};
struct PassThroughExec : Operator {   // CoalesceBatches / BroadcastJoinBuildHashMap / Debug: batch shape is not part of the contract
    PassThroughExec(OperatorPtr input, const std::string& nm);
    BatchPtr next(Task& t) override { return children[0]->next(t); }
};
// expand_exec.rs:127-185: every input batch is emitted once per projection list (GROUPING SETS / ROLLUP / CUBE), each expression
// cast to the declared output field type
struct ExpandExec : Operator {
    std::vector<std::vector<ExprPtr>> projections;
    std::vector<VmProgram> progs;
    std::vector<std::vector<int>> plain;   // per projection, per output column: >= 0 bare input column, -1 computed (next program output)
    BatchPtr cur;
    size_t next_proj = 0;
    ExpandExec(OperatorPtr input, const Schema& schema, std::vector<std::vector<ExprPtr>> projections);
    std::string describe() const override;
    BatchPtr next(Task& t) override;
};

// generate_exec.rs:120-310 + generate/explode.rs: explode / posexplode of a list column, with or without `outer`.  The input comes
// through next_sel (a Filter below hands over its selection); the output of one input batch is cut between input rows into
// pieces of at most gpu_chunk_rows rows whose string columns stay addressable with int32 offsets.
enum GenerateFn { GEN_EXPLODE = 0, GEN_POS_EXPLODE = 1 };
struct GenerateExec : Operator {
    int func = GEN_EXPLODE;
    bool outer = false;
    std::vector<int> required;            // input columns copied once per output row
    std::vector<std::string> required_names;
    std::vector<Field> gen_fields;        // [pos int32,] element
    ListExpr gen;
    VmProgram prog;                       // flat arguments of gen
    bool has_prog = false;
    // the input batch being exploded (one at a time)
    SelBatch cur;
    ColumnPtr list;
    Buf rows_cum, bytes_cum;
    int64_t next_row = 0;
    GenerateExec(OperatorPtr input, int func, const ExprPtr& child, std::vector<std::string> required, std::vector<Field> gen_output, bool outer);
    std::string describe() const override;
    BatchPtr next(Task& t) override;
};

// union_exec.rs:118-160
struct UnionExec : Operator {
    size_t cur = 0;
    UnionExec(std::vector<OperatorPtr> inputs, const Schema& schema);
    BatchPtr next(Task& t) override;
};

// helpers shared with scan / shuffle
ColumnPtr eval_to_column(Task& t, const ExprPtr& e, const Schema& schema, const Batch& b);
BatchPtr materialize(Task& t, SelBatch& s);

}  // namespace auron
