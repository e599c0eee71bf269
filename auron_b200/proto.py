"""Hand-written proto3 encoder for the subset of Auron's plan wire format (auron.proto) on the hot path.

This is the caller side of the boundary: what Spark's NativeConverters / Native*Base classes
(spark-extension/src/main/scala/org/apache/spark/sql/auron/NativeConverters.scala:400-1300,
.../execution/auron/plan/Native*Base.scala) emit per stage.  No protoc exists in this image, so the
messages are encoded by field number (native-engine/auron-planner/proto/auron.proto).  Every builder
returns the serialized bytes of the message named in its docstring.
"""
from __future__ import annotations

import pyarrow as pa


def _varint(n: int) -> bytes:
    if n < 0:
        n += 1 << 64
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def f_varint(num: int, v: int, always: bool = False) -> bytes:
    """proto3 scalar field: a zero value is NOT written (protobuf-java and prost both omit default-valued scalars), so the
    planner's defaults are exercised the way real plans exercise them.  `always` is for oneof members and packed elements."""
    if int(v) == 0 and not always:
        return b""
    return _varint(num << 3) + _varint(int(v))


def f_bytes(num: int, b: bytes) -> bytes:
    return _varint((num << 3) | 2) + _varint(len(b)) + b


def f_str(num: int, s: str) -> bytes:
    return f_bytes(num, s.encode())


# ----------------------------------------------------------------------------- types / schema
def arrow_type(t: pa.DataType) -> bytes:
    """ArrowType (auron.proto:915-951)"""
    empty = b""
    if pa.types.is_null(t):
        return f_bytes(1, empty)
    if pa.types.is_boolean(t):
        return f_bytes(2, empty)
    if pa.types.is_int8(t):
        return f_bytes(4, empty)
    if pa.types.is_int16(t):
        return f_bytes(6, empty)
    if pa.types.is_int32(t):
        return f_bytes(8, empty)
    if pa.types.is_int64(t):
        return f_bytes(10, empty)
    if pa.types.is_float32(t):
        return f_bytes(12, empty)
    if pa.types.is_float64(t):
        return f_bytes(13, empty)
    if pa.types.is_string(t):
        return f_bytes(14, empty)
    if pa.types.is_binary(t):
        return f_bytes(15, empty)
    if pa.types.is_date32(t):
        return f_bytes(17, empty)
    if pa.types.is_date64(t):
        return f_bytes(18, empty)
    if pa.types.is_timestamp(t):
        unit = {"s": 0, "ms": 1, "us": 2, "ns": 3}[t.unit]
        body = f_varint(1, unit) + (f_str(2, t.tz) if t.tz else b"")
        return f_bytes(20, body)
    if pa.types.is_decimal128(t):
        return f_bytes(24, f_varint(1, t.precision) + f_varint(2, t.scale))
    if pa.types.is_list(t):
        return f_bytes(25, f_bytes(1, field(t.value_field.name, t.value_type, t.value_field.nullable)))   # List{field_type}
    raise NotImplementedError(str(t))


def field(name: str, t: pa.DataType, nullable: bool = True) -> bytes:
    """Field (auron.proto:805-810)"""
    return f_str(1, name) + f_bytes(2, arrow_type(t)) + f_varint(3, 1 if nullable else 0)


def schema(s: pa.Schema) -> bytes:
    """Schema (auron.proto:801-803)"""
    return b"".join(f_bytes(1, field(f.name, f.type, f.nullable)) for f in s)


# ----------------------------------------------------------------------------- expressions
def scalar_value(value, t: pa.DataType) -> bytes:
    """ScalarValue{ipc_bytes}: an Arrow IPC stream with a 1-row, 1-column batch (NativeConverters.scala:413-428)"""
    arr = pa.array([value], type=t)
    batch = pa.record_batch([arr], names=["v"])
    sink = pa.BufferOutputStream()
    with pa.ipc.new_stream(sink, batch.schema) as w:
        w.write_batch(batch)
    return f_bytes(1, sink.getvalue().to_pybytes())


def col(name: str, index: int = 0) -> bytes:
    """PhysicalExprNode{column}"""
    return f_bytes(1, f_str(1, name) + f_varint(2, index))


def bound_ref(index: int, t: pa.DataType, nullable: bool = True) -> bytes:
    return f_bytes(3, f_varint(1, index) + f_bytes(2, arrow_type(t)) + f_varint(3, int(nullable)))


def lit(value, t: pa.DataType) -> bytes:
    """PhysicalExprNode{literal}"""
    return f_bytes(2, scalar_value(value, t))


def binary(op: str, l: bytes, r: bytes) -> bytes:
    """PhysicalExprNode{binary_expr{l,r,op}} -- op names per auron-planner/src/lib.rs:70-101"""
    return f_bytes(4, f_bytes(1, l) + f_bytes(2, r) + f_str(3, op))


def is_null(e: bytes) -> bytes:
    return f_bytes(6, f_bytes(1, e))


def is_not_null(e: bytes) -> bytes:
    return f_bytes(7, f_bytes(1, e))


def not_(e: bytes) -> bytes:
    return f_bytes(8, f_bytes(1, e))


def negative(e: bytes) -> bytes:
    return f_bytes(12, f_bytes(1, e))


def case(when_then: list[tuple[bytes, bytes]], else_expr: bytes | None = None, expr: bytes | None = None) -> bytes:
    body = b""
    if expr is not None:
        body += f_bytes(1, expr)
    for w, t in when_then:
        body += f_bytes(2, f_bytes(1, w) + f_bytes(2, t))
    if else_expr is not None:
        body += f_bytes(3, else_expr)
    return f_bytes(9, body)


def cast(e: bytes, t: pa.DataType) -> bytes:
    return f_bytes(10, f_bytes(1, e) + f_bytes(2, arrow_type(t)))


def try_cast(e: bytes, t: pa.DataType) -> bytes:
    return f_bytes(15, f_bytes(1, e) + f_bytes(2, arrow_type(t)))


def in_list(e: bytes, items: list[bytes], negated: bool = False) -> bytes:
    return f_bytes(13, f_bytes(1, e) + b"".join(f_bytes(2, i) for i in items) + f_varint(3, int(negated)))


SCALAR_FN = {"Abs": 0, "Ascii": 4, "Ceil": 5, "Exp": 8, "Floor": 9, "Ln": 10, "Log10": 12, "Log2": 13, "Signum": 15, "Sqrt": 17,
             "NullIf": 20, "BitLength": 22, "CharacterLength": 24, "Chr": 25, "DatePart": 28, "DateTrunc": 29, "Lpad": 32, "Lower": 33,
             "Ltrim": 34, "OctetLength": 37, "Replace": 41, "Reverse": 42, "Rpad": 44, "Rtrim": 45, "StartsWith": 51, "Substr": 53,
             "Translate": 60, "Trim": 61, "Upper": 62, "Coalesce": 63, "Factorial": 65, "Hex": 66, "Power": 67, "Acosh": 68, "IsNaN": 69,
             "Levenshtein": 80, "FindInSet": 81, "Nvl2": 83, "Least": 84, "Greatest": 85, "MakeDate": 86, "AuronExtFunctions": 10000}


def scalar_fn(name: str, args: list[bytes], return_type: pa.DataType) -> bytes:
    """PhysicalExprNode{scalar_function{name, fun, args, return_type}}; unknown names go through AuronExtFunctions"""
    fun = SCALAR_FN.get(name, 10000)
    return f_bytes(14, f_str(1, name) + f_varint(2, fun) + b"".join(f_bytes(3, a) for a in args) + f_bytes(4, arrow_type(return_type)))


def like(e: bytes, pattern: bytes, negated: bool = False, case_insensitive: bool = False) -> bytes:
    return f_bytes(20, f_varint(1, int(negated)) + f_varint(2, int(case_insensitive)) + f_bytes(3, e) + f_bytes(4, pattern))


def sc_and(l: bytes, r: bytes) -> bytes:
    return f_bytes(3000, f_bytes(1, l) + f_bytes(2, r))


def sc_or(l: bytes, r: bytes) -> bytes:
    return f_bytes(3001, f_bytes(1, l) + f_bytes(2, r))


def starts_with(e: bytes, prefix: str) -> bytes:
    return f_bytes(20000, f_bytes(1, e) + f_str(2, prefix))


def ends_with(e: bytes, suffix: str) -> bytes:
    return f_bytes(20001, f_bytes(1, e) + f_str(2, suffix))


def contains(e: bytes, infix: str) -> bytes:
    return f_bytes(20002, f_bytes(1, e) + f_str(2, infix))


def row_num() -> bytes:
    """PhysicalExprNode{row_num_expr} (NativeConverters.scala StubExpr("RowNum"))"""
    return f_bytes(20100, b"")


def spark_partition_id() -> bytes:
    """PhysicalExprNode{spark_partition_id_expr}"""
    return f_bytes(20101, b"")


AGG_FN = {"MIN": 0, "MAX": 1, "SUM": 2, "AVG": 3, "COUNT": 4, "FIRST": 7, "FIRST_IGNORES_NULL": 8}
AGG_MODE = {"PARTIAL": 0, "PARTIAL_MERGE": 1, "FINAL": 2}


def agg_expr(fn: str, children: list[bytes], return_type: pa.DataType) -> bytes:
    """PhysicalExprNode{agg_expr{agg_function, children, return_type}}"""
    return f_bytes(5, f_varint(1, AGG_FN[fn]) + b"".join(f_bytes(3, c) for c in children) + f_bytes(4, arrow_type(return_type)))


def sort_expr(e: bytes, asc: bool = True, nulls_first: bool = True) -> bytes:
    """PhysicalExprNode{sort{expr, asc, nulls_first}}"""
    return f_bytes(11, f_bytes(1, e) + f_varint(2, int(asc)) + f_varint(3, int(nulls_first)))


# ----------------------------------------------------------------------------- plan nodes
def ffi_reader(s: pa.Schema, resource_id: str, num_partitions: int = 1) -> bytes:
    """PhysicalPlanNode{ffi_reader} (ConvertToNativeBase.scala:82)"""
    return f_bytes(18, f_varint(1, num_partitions) + f_bytes(2, schema(s)) + f_str(3, resource_id))


def ipc_reader(s: pa.Schema, resource_id: str, num_partitions: int = 1) -> bytes:
    """PhysicalPlanNode{ipc_reader}: shuffle read (auron.proto:636-640)"""
    return f_bytes(3, f_varint(1, num_partitions) + f_bytes(2, schema(s)) + f_str(3, resource_id))


def filter_(inp: bytes, exprs: list[bytes]) -> bytes:
    return f_bytes(8, f_bytes(1, inp) + b"".join(f_bytes(2, e) for e in exprs))


def projection(inp: bytes, exprs: list[bytes], names: list[str], types: list[pa.DataType]) -> bytes:
    return f_bytes(6, f_bytes(1, inp) + b"".join(f_bytes(2, e) for e in exprs) + b"".join(f_str(3, n) for n in names)
                   + b"".join(f_bytes(4, arrow_type(t)) for t in types))


def agg(inp: bytes, grouping: list[bytes], grouping_names: list[str], aggs: list[bytes], agg_names: list[str], modes: list[str],
        exec_mode: int = 0, supports_partial_skipping: bool = False) -> bytes:
    """PhysicalPlanNode{agg} (NativeAggBase.scala:190)"""
    body = f_bytes(1, inp) + f_varint(2, exec_mode)
    body += b"".join(f_bytes(3, g) for g in grouping)
    body += b"".join(f_bytes(4, a) for a in aggs)
    body += b"".join(f_varint(5, AGG_MODE[m], always=True) for m in modes)   # repeated: every element is written
    body += b"".join(f_str(6, n) for n in grouping_names)
    body += b"".join(f_str(7, n) for n in agg_names)
    body += f_varint(9, int(supports_partial_skipping))
    return f_bytes(16, body)


JOIN_TYPE = {"INNER": 0, "LEFT": 1, "RIGHT": 2, "FULL": 3, "SEMI": 4, "ANTI": 5, "EXISTENCE": 6}


def _join_on(on: list[tuple[bytes, bytes]]) -> bytes:
    return b"".join(f_bytes(4, f_bytes(1, l) + f_bytes(2, r)) for l, r in on)


def hash_join(s: pa.Schema, left: bytes, right: bytes, on: list[tuple[bytes, bytes]], join_type: str, build_side: str) -> bytes:
    """PhysicalPlanNode{hash_join} (NativeShuffledHashJoinBase.scala:134)"""
    return f_bytes(11, f_bytes(1, schema(s)) + f_bytes(2, left) + f_bytes(3, right) + _join_on(on) + f_varint(5, JOIN_TYPE[join_type])
                   + f_varint(6, 0 if build_side == "LEFT" else 1))


def sort_merge_join(s: pa.Schema, left: bytes, right: bytes, on: list[tuple[bytes, bytes]], join_type: str) -> bytes:
    """PhysicalPlanNode{sort_merge_join} (NativeSortMergeJoinBase.scala:153)"""
    opts = b"".join(f_bytes(5, f_varint(1, 1) + f_varint(2, 1)) for _ in on)
    return f_bytes(10, f_bytes(1, schema(s)) + f_bytes(2, left) + f_bytes(3, right) + _join_on(on) + opts + f_varint(6, JOIN_TYPE[join_type]))


def broadcast_join(s: pa.Schema, left: bytes, right: bytes, on: list[tuple[bytes, bytes]], join_type: str, broadcast_side: str,
                   cached_id: str = "", null_aware_anti: bool = False) -> bytes:
    return f_bytes(13, f_bytes(1, schema(s)) + f_bytes(2, left) + f_bytes(3, right) + _join_on(on) + f_varint(5, JOIN_TYPE[join_type])
                   + f_varint(6, 0 if broadcast_side == "LEFT" else 1) + f_str(7, cached_id) + f_varint(8, int(null_aware_anti)))


def sort(inp: bytes, sort_exprs: list[bytes], limit: int | None = None, offset: int = 0) -> bytes:
    body = f_bytes(1, inp) + b"".join(f_bytes(2, e) for e in sort_exprs)
    if limit is not None:
        body += f_bytes(3, f_varint(1, limit) + f_varint(2, offset))
    return f_bytes(7, body)


def limit(inp: bytes, n: int, offset: int = 0) -> bytes:
    return f_bytes(17, f_bytes(1, inp) + f_varint(2, n) + f_varint(3, offset))


def rename_columns(inp: bytes, names: list[str]) -> bytes:
    return f_bytes(14, f_bytes(1, inp) + b"".join(f_str(2, n) for n in names))


def union(inputs: list[bytes], s: pa.Schema) -> bytes:
    return f_bytes(9, b"".join(f_bytes(1, f_bytes(1, i) + f_varint(2, 0)) for i in inputs) + f_bytes(2, schema(s)) + f_varint(3, 1))


def expand(inp: bytes, s: pa.Schema, projections: list[list[bytes]]) -> bytes:
    """PhysicalPlanNode{expand{input, schema, projections{expr}}} (auron.proto:745-754)"""
    body = f_bytes(1, inp) + f_bytes(2, schema(s)) + b"".join(f_bytes(3, b"".join(f_bytes(1, e) for e in pr)) for pr in projections)
    return f_bytes(20, body)


WINDOW_FUNCTION = {"ROW_NUMBER": 0, "RANK": 1, "DENSE_RANK": 2, "LEAD": 3, "NTH_VALUE": 4, "NTH_VALUE_IGNORE_NULLS": 5, "PERCENT_RANK": 6, "CUME_DIST": 7}


def window_expr(name: str, t: pa.DataType, fn: str, children: list[bytes] | None = None) -> bytes:
    """WindowExprNode{field=1, return_type=1000, func_type=2, window_func=3, agg_func=4, children=5} (auron.proto:575-582); fn is a
    WindowFunction name or an AggFunction name"""
    body = f_bytes(1, field(name, t)) + f_bytes(1000, arrow_type(t))
    if fn in WINDOW_FUNCTION:
        body += f_varint(2, 0) + f_varint(3, WINDOW_FUNCTION[fn])
    else:
        body += f_varint(2, 1) + f_varint(4, AGG_FN[fn])
    return body + b"".join(f_bytes(5, c) for c in (children or []))


def window(inp: bytes, window_exprs: list[bytes], partition_spec: list[bytes], order_spec: list[bytes], group_limit: int | None = None,
           output_window_cols: bool = True) -> bytes:
    """PhysicalPlanNode{window} (auron.proto:566-573); order_spec entries are sort expressions (sort_expr)"""
    body = f_bytes(1, inp) + b"".join(f_bytes(2, w) for w in window_exprs) + b"".join(f_bytes(3, e) for e in partition_spec) + b"".join(f_bytes(4, e) for e in order_spec)
    if group_limit is not None:
        body += f_bytes(5, f_varint(1, group_limit, always=True))
    return f_bytes(22, body + f_varint(6, int(output_window_cols)))


GENERATE_FUNCTION = {"Explode": 0, "PosExplode": 1, "JsonTuple": 2, "Udtf": 10000}


def generate(inp: bytes, func: str, child: bytes, required_child_output: list[str], generator_output: list[tuple[str, pa.DataType, bool]],
             outer: bool = False) -> bytes:
    """PhysicalPlanNode{generate{input, generator{func, child}, required_child_output, generator_output, outer}} (auron.proto:593-612;
    NativeGenerateBase.scala); generator_output holds (name, type, nullable) per generated column"""
    gen = f_varint(1, GENERATE_FUNCTION[func]) + f_bytes(3, child)
    body = f_bytes(1, inp) + f_bytes(2, gen) + b"".join(f_str(3, n) for n in required_child_output)
    body += b"".join(f_bytes(4, field(n, t, nl)) for n, t, nl in generator_output)
    return f_bytes(23, body + f_varint(5, int(outer)))


def ipc_writer(inp: bytes, consumer_resource_id: str) -> bytes:
    """PhysicalPlanNode{ipc_writer{input, ipc_consumer_resource_id}} (auron.proto:631-634; NativeBroadcastExchangeBase.scala:317-328)"""
    return f_bytes(4, f_bytes(1, inp) + f_str(2, consumer_resource_id))


def hash_repartition(exprs: list[bytes], n: int) -> bytes:
    """PhysicalRepartition{hash_repartition}"""
    return f_bytes(2, b"".join(f_bytes(1, e) for e in exprs) + f_varint(2, n))


def single_repartition(n: int = 1) -> bytes:
    return f_bytes(1, f_varint(1, n))


def round_robin_repartition(n: int) -> bytes:
    return f_bytes(3, f_varint(1, n))


def range_repartition(sort_exprs: list[bytes], n: int, bounds: list[tuple[list, pa.DataType]]) -> bytes:
    """PhysicalRepartition{range_repartition}: sort expressions (inside a SortExecNode without input), partition count and one
    List ScalarValue of n - 1 bound values per sort expression (auron.proto:681-685, planner.rs:1160-1210)"""
    sort_node = b"".join(f_bytes(2, e) for e in sort_exprs)
    return f_bytes(4, f_bytes(1, sort_node) + f_varint(2, n) + b"".join(f_bytes(3, scalar_value(vals, pa.list_(t))) for vals, t in bounds))


def shuffle_writer(inp: bytes, repartition: bytes, data_file: str, index_file: str) -> bytes:
    """PhysicalPlanNode{shuffle_writer} (auron.proto:553-558)"""
    return f_bytes(2, f_bytes(1, inp) + f_bytes(2, repartition) + f_str(3, data_file) + f_str(4, index_file))


def parquet_scan(s: pa.Schema, files: list[tuple[str, int]], projection_idx: list[int], fs_resource_id: str = "",
                 pruning_predicates: list[bytes] | None = None, ranges: list[tuple[int, int]] | None = None,
                 partition_schema: pa.Schema | None = None, partition_values: list[list] | None = None) -> bytes:
    """PhysicalPlanNode{parquet_scan{base_conf{...}, pruning_predicates, fsResourceId}} (NativeParquetScanBase.scala:73-85).
    partition_schema / partition_values: Hive partition columns (NativeFileSourceScanBase.scala:105-129): one value per partition
    column and file; projection indices >= len(s) address them."""
    pfiles = b""
    for i, (path, size) in enumerate(files):
        pf = f_str(1, path) + f_varint(2, size)
        if partition_schema is not None:
            for fld, v in zip(partition_schema, partition_values[i]):
                pf += f_bytes(4, scalar_value(v, fld.type))
        if ranges is not None:
            pf += f_bytes(5, f_varint(1, ranges[i][0]) + f_varint(2, ranges[i][1]))
        pfiles += f_bytes(1, pf)
    conf = f_varint(1, 1) + f_varint(2, 0) + f_bytes(3, pfiles) + f_bytes(4, schema(s))
    conf += b"".join(f_varint(6, p, always=True) for p in projection_idx)   # repeated
    if partition_schema is not None:
        conf += f_bytes(9, schema(partition_schema))
    body = f_bytes(1, conf) + b"".join(f_bytes(2, p) for p in (pruning_predicates or [])) + f_str(3, fs_resource_id)
    return f_bytes(5, body)


def task_definition(plan: bytes, stage_id: int = 0, partition_id: int = 0, task_id: int = 0) -> bytes:
    """TaskDefinition{task_id: PartitionId, plan} (auron.proto:784-795)"""
    pid = f_varint(2, stage_id) + f_varint(4, partition_id) + f_varint(5, task_id)
    return f_bytes(1, pid) + f_bytes(2, plan)
