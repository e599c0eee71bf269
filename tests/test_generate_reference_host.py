"""CPU checks of explode / posexplode, split and array(): generate_reference.py against the reference's own goldens, and the planner
(through runtime.explain) on every accepted and rejected shape of generate and list columns."""
import pyarrow as pa
import pytest

from auron_b200 import proto as P
from auron_b200 import runtime
from generate_reference import explode, list_offsets, make_array, string_split

U = pa.string()
LU = pa.list_(pa.string())
LI = pa.list_(pa.int32())
T = pa.schema([("a", pa.int32()), ("s", U), ("l", LI), ("ls", LU)])


# ----------------------------------------------------------------------------- the reference's goldens
def test_string_split_golden():
    # spark_strings.rs:448-481 (test_string_split)
    lists = [string_split(s, ",") for s in ["123,456,,,789,", "123", "", None]]
    assert list_offsets(lists) == [0, 6, 7, 8, 8]
    assert [v for lst in lists if lst for v in lst] == ["123", "456", "", "", "789", "", "123", ""]
    assert lists[3] is None


def test_string_split_edges():
    assert string_split("---", "--") == ["", "-"]           # leftmost, non-overlapping
    assert string_split(",a,", ",") == ["", "a", ""]
    assert string_split("a<>b<>", "<>") == ["a", "b", ""]
    assert string_split("añb", "ñ") == ["a", "b"]


def test_make_array_golden():
    # spark_make_array.rs:155-218
    col = [12, -123, 0, 9, None]
    assert make_array(col) == [[12], [-123], [0], [9], [None]]
    assert make_array([123456] * 5, col) == [[123456, 12], [123456, -123], [123456, 0], [123456, 9], [123456, None]]
    assert make_array([2.2], [-2.3]) == [[2.2, -2.3]]


def test_explode_golden():
    # generate_exec.rs:373-530 (test_explode): a, b = [[400, 500, NULL], [600, 700, 800], [], NULL]
    a = [(1,), (2,), (3,), (None,)]
    b = [[400, 500, None], [600, 700, 800], [], None]
    assert explode(a, b) == [(1, 400), (1, 500), (1, None), (2, 600), (2, 700), (2, 800)]
    assert explode(a, b, outer=True) == [(1, 400), (1, 500), (1, None), (2, 600), (2, 700), (2, 800), (3, None), (None, None)]
    assert explode(a, b, pos=True, outer=True) == [(1, 0, 400), (1, 1, 500), (1, 2, None), (2, 0, 600), (2, 1, 700), (2, 2, 800),
                                                   (3, None, None), (None, None, None)]


# ----------------------------------------------------------------------------- planning
def _explain(plan):
    return runtime.explain(P.task_definition(plan))["plan"]


def _error(plan) -> str:
    with pytest.raises(runtime.AuronError) as e:
        runtime.explain(P.task_definition(plan))
    return str(e.value)


SRC = P.ffi_reader(T, "t")
SPLIT = P.scalar_fn("Spark_StringSplit", [P.col("s"), P.lit(",", U)], LU)
ARRAY = P.scalar_fn("Spark_MakeArray", [P.col("a"), P.lit(7, pa.int32())], LI)


def test_list_columns_and_expressions_are_projected():
    d = _explain(P.projection(SRC, [P.col("l"), SPLIT, ARRAY, P.lit([1, None], LI)], ["l", "p", "arr", "k"], [LI, LU, LI, LI]))
    assert d["op"] == "ProjectExec"
    assert d["schema"] == [["l", "list<int32>"], ["p", "list<utf8>"], ["arr", "list<int32>"], ["k", "list<int32>"]]
    assert d["children"][0]["schema"][2:] == [["l", "list<int32>"], ["ls", "list<utf8>"]]


@pytest.mark.parametrize("func,outer", [("Explode", False), ("Explode", True), ("PosExplode", False), ("PosExplode", True)])
def test_generate_is_planned(func, outer):
    gout = ([("pos", pa.int32(), False)] if func == "PosExplode" else []) + [("w", U, True)]
    d = _explain(P.generate(P.projection(SRC, [P.col("a"), SPLIT], ["a", "parts"], [pa.int32(), LU]), func, P.col("parts"), ["a"], gout, outer))
    assert (d["op"], d["function"], d["outer"], d["required"], d["child"]) == ("GenerateExec", func, outer, ["a"], "col(parts)")
    assert d["schema"] == [["a", "int32"]] + ([["pos", "int32"]] if func == "PosExplode" else []) + [["w", "utf8"]]


def test_generate_child_shapes_and_required_orders():
    for child, et in ((SPLIT, "utf8"), (ARRAY, "int32"), (P.lit([1, 2], LI), "int32"), (P.col("l"), "int32")):
        t = pa.string() if et == "utf8" else pa.int32()
        for req in ([], ["s"], ["s", "a"]):
            d = _explain(P.generate(SRC, "Explode", child, req, [("v", t, True)]))
            assert [f[0] for f in d["schema"]] == req + ["v"] and d["schema"][-1][1] == et


def test_list_columns_pass_through_the_carrying_operators():
    flt = P.filter_(SRC, [P.binary("Gt", P.col("a"), P.lit(0, pa.int32()))])
    for plan, op in ((flt, "FilterExec"), (P.limit(SRC, 3), "LimitExec"), (P.union([SRC, SRC], T), "UnionExec"),
                     (P.rename_columns(SRC, ["x", "y", "z", "w"]), "RenameColumnsExec"), (P.f_bytes(19, P.f_bytes(1, SRC)), "CoalesceBatchesExec")):
        d = _explain(plan)
        assert d["op"] == op and d["schema"][2][1] == "list<int32>"


REJECTED_EXPR = {
    "split_in_function": ("Spark_StringSplit", P.projection(SRC, [P.scalar_fn("Upper", [SPLIT], U)], ["x"], [U])),
    "split_in_case": ("Spark_StringSplit", P.projection(SRC, [P.case([(P.is_null(P.col("a")), SPLIT)], SPLIT)], ["x"], [LU])),
    "cast_of_list": ("Cast(", P.projection(SRC, [P.cast(P.col("l"), LU)], ["x"], [LU])),
    "list_in_predicate": ("list column l", P.filter_(SRC, [P.is_null(P.col("l"))])),
    "split_in_predicate": ("Spark_StringSplit", P.filter_(SRC, [P.is_not_null(SPLIT)])),
    "non_literal_pattern": ("Spark_StringSplit", P.projection(SRC, [P.scalar_fn("Spark_StringSplit", [P.col("s"), P.col("s")], LU)], ["x"], [LU])),
    "empty_pattern": ("Spark_StringSplit", P.projection(SRC, [P.scalar_fn("Spark_StringSplit", [P.col("s"), P.lit("", U)], LU)], ["x"], [LU])),
    "mixed_array": ("Spark_MakeArray", P.projection(SRC, [P.scalar_fn("Spark_MakeArray", [P.col("a"), P.col("s")], LI)], ["x"], [LI])),
    "split_as_agg_key": ("Spark_StringSplit", P.agg(SRC, [SPLIT], ["k"], [P.agg_expr("COUNT", [P.col("a")], pa.int64())], ["c"], ["PARTIAL"])),
    "split_as_sort_key": ("Spark_StringSplit", P.sort(P.projection(SRC, [P.col("a"), P.col("s")], ["a", "s"], [pa.int32(), U]), [P.sort_expr(SPLIT)])),
    "split_as_shuffle_key": ("Spark_StringSplit", P.shuffle_writer(P.projection(SRC, [P.col("s")], ["s"], [U]), P.hash_repartition([SPLIT], 4), "/tmp/d", "/tmp/i")),
}


@pytest.mark.parametrize("case", sorted(REJECTED_EXPR))
def test_list_expressions_outside_their_places_are_rejected_by_name(case):
    needle, plan = REJECTED_EXPR[case]
    assert needle in _error(plan)


def _agg(src, key):
    return P.agg(src, [P.col(key)], [key], [P.agg_expr("COUNT", [P.col("a")], pa.int64())], ["c"], ["PARTIAL"])


REJECTED_OP = {
    "sort": ("SortExec", P.sort(SRC, [P.sort_expr(P.col("a"))])),
    "agg_key": ("AggExec", _agg(SRC, "l")),
    "agg_arg": ("AggExec", P.agg(SRC, [P.col("a")], ["a"], [P.agg_expr("COUNT", [P.col("ls")], pa.int64())], ["c"], ["PARTIAL"])),
    "hash_join": ("HashJoinExec", P.hash_join(pa.schema(list(T) + list(T)), SRC, SRC, [(P.col("a"), P.col("a"))], "INNER", "RIGHT")),
    "smj": ("SortMergeJoinExec", P.sort_merge_join(pa.schema(list(T) + list(T)), SRC, SRC, [(P.col("a"), P.col("a"))], "INNER")),
    "bhj": ("BroadcastJoinExec", P.broadcast_join(pa.schema(list(T) + list(T)), SRC, SRC, [(P.col("a"), P.col("a"))], "INNER", "RIGHT")),
    "window": ("WindowExec", P.window(SRC, [P.window_expr("r", pa.int32(), "ROW_NUMBER")], [P.col("a")], [P.sort_expr(P.col("a"))])),
    "expand": ("ExpandExec", P.expand(SRC, T, [[P.col("a"), P.col("s"), P.col("l"), P.col("ls")]])),
    "shuffle": ("ShuffleWriterExec", P.shuffle_writer(SRC, P.hash_repartition([P.col("a")], 4), "/tmp/d", "/tmp/i")),
    "ipc_writer": ("IpcWriterExec", P.ipc_writer(SRC, "c")),
    "ipc_reader": ("IpcReaderExec", P.ipc_reader(T, "blocks")),
}


@pytest.mark.parametrize("case", sorted(REJECTED_OP))
def test_operators_that_cannot_carry_lists_name_the_operator_and_column(case):
    op, plan = REJECTED_OP[case]
    msg = _error(plan)
    assert op in msg and ("list column l " in msg or "list column ls " in msg), msg


def test_generate_rejections():
    gout = [("v", pa.int32(), True)]
    assert "not native" in _error(P.generate(SRC, "JsonTuple", P.col("s"), [], [("v", U, True)]))
    assert "not native" in _error(P.generate(SRC, "Udtf", P.col("s"), [], [("v", U, True)]))
    assert "not native" in _error(P.f_bytes(23, P.f_bytes(1, SRC)))
    assert "not native" in _error(P.generate(SRC, "Explode", P.col("a"), [], gout))                       # not a list
    assert "value column v must be utf8" in _error(P.generate(SRC, "Explode", SPLIT, [], gout))             # element type mismatch
    assert "position column" in _error(P.generate(SRC, "PosExplode", P.col("l"), [], [("p", pa.int64(), True), ("v", pa.int32(), True)]))
    assert "produces 2 columns" in _error(P.generate(SRC, "PosExplode", P.col("l"), [], gout))
    assert "nope" in _error(P.generate(SRC, "Explode", P.col("l"), ["nope"], gout))
    assert "not native" in _error(P.agg(SRC, [P.col("a")], ["a"], [P.f_bytes(5, P.f_varint(1, 5) + P.f_bytes(3, P.col("a")) + P.f_bytes(4, P.arrow_type(LI)))],
                                        ["c"], ["PARTIAL"]))   # COLLECT_LIST


def test_nested_types_other_than_one_list_level_stay_rejected():
    field = lambda t: P.f_str(1, "x") + P.f_bytes(2, t) + P.f_varint(3, 1)
    large = P.f_bytes(26, P.f_bytes(1, P.field("item", pa.int32())))
    list_of_list = P.f_bytes(25, P.f_bytes(1, P.field("item", LI)))
    struct = P.f_bytes(28, P.f_bytes(1, P.field("f", pa.int32())))
    for t, needle in ((large, "tag 26"), (list_of_list, "list of list"), (struct, "struct")):
        src = P.f_bytes(18, P.f_varint(1, 1) + P.f_bytes(2, P.f_bytes(1, field(t))) + P.f_str(3, "t"))
        msg = _error(src)
        assert needle in msg and "nested types are out of scope" in msg, msg
