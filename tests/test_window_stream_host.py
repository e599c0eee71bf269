"""CPU checks of the window aggregates' argument types: the planner, through runtime.explain, accepts every SUM / AVG / MIN / MAX
shape the engine computes on the device and rejects the others when the plan is built, with a message that names the function and
the type.

Argument types restated from the reference (native-engine/datafusion-ext-plans/src/agg): SUM / AVG over numbers and decimals
(sum.rs, avg.rs; the argument is cast to the declared result type first, agg.rs:191-198), MIN / MAX over any primitive, decimal,
utf8 or binary value (maxmin.rs), COUNT over anything (count.rs).
"""
import pyarrow as pa
import pytest

from auron_b200 import proto as P
from auron_b200 import runtime

T = pa.schema([("p", pa.int32()), ("o", pa.int64()), ("d17", pa.decimal128(17, 2)), ("d21", pa.decimal128(21, 6)), ("d38", pa.decimal128(38, 10)),
               ("s", pa.string()), ("b", pa.binary()), ("f", pa.bool_()), ("ts", pa.timestamp("us")), ("tn", pa.timestamp("ns", tz="UTC")),
               ("d64", pa.date64()), ("i", pa.int64())])


def _plan(wex):
    src = P.ffi_reader(T, "t")
    return P.task_definition(P.window(src, wex, [P.col("p")], [P.sort_expr(P.col("o"))]))


def _error(wex) -> str:
    with pytest.raises(runtime.AuronError) as e:
        runtime.explain(_plan(wex))
    return str(e.value)


def test_new_window_aggregate_shapes_are_planned():
    wex = [P.window_expr("sum17", pa.decimal128(27, 2), "SUM", [P.col("d17")]),
           P.window_expr("avg21", pa.decimal128(25, 10), "AVG", [P.col("d21")]),
           P.window_expr("min38", pa.decimal128(38, 10), "MIN", [P.col("d38")]),
           P.window_expr("max38", pa.decimal128(38, 10), "MAX", [P.col("d38")])]
    names = ["sum17", "avg21", "min38", "max38"]
    for c, t in (("s", pa.string()), ("b", pa.binary()), ("f", pa.bool_()), ("ts", pa.timestamp("us")), ("tn", pa.timestamp("ns", tz="UTC")),
                 ("d64", pa.date64())):
        for fn in ("MIN", "MAX"):
            wex.append(P.window_expr(f"{fn.lower()}_{c}", t, fn, [P.col(c)]))
            names.append(f"{fn.lower()}_{c}")
    d = runtime.explain(_plan(wex))["plan"]
    assert d["op"] == "WindowExec"
    fns = [x.split(" AS ") for x in d["functions"]]
    assert [n for _, n in fns] == names
    assert [f for f, _ in fns] == ["SUM", "AVG", "MIN", "MAX"] + ["MIN", "MAX"] * 6
    assert [f[0] for f in d["schema"]] == list(T.names) + names


def test_sum_and_avg_over_decimals_cast_like_the_aggregate():
    # AVG over decimal(21,6) returning decimal(25,10): the argument is cast to the result type (scale 6 -> 10) before the running
    # sum; SUM over decimal(17,2) returning decimal(27,2) keeps the scale and needs no cast
    wex = [P.window_expr("a", pa.decimal128(25, 10), "AVG", [P.col("d21")]), P.window_expr("s", pa.decimal128(27, 2), "SUM", [P.col("d17")])]
    d = runtime.explain(_plan(wex))["plan"]
    assert d["functions"] == ["AVG AS a", "SUM AS s"]
    assert [f[1] for f in d["schema"][-2:]] == ["decimal128(25,10)", "decimal128(27,2)"]


@pytest.mark.parametrize("fn,col,ret,type_name", [("SUM", "s", pa.string(), "utf8"), ("AVG", "f", pa.float64(), "bool"),
                                                   ("SUM", "b", pa.binary(), "binary"), ("AVG", "ts", pa.float64(), "timestamp")])
def test_unsupported_argument_types_are_rejected_by_name(fn, col, ret, type_name):
    msg = _error([P.window_expr("w", ret, fn, [P.col(col)])])
    assert f"window {fn} over {type_name}" in msg and "not supported" in msg


def test_min_over_a_list_is_rejected_by_name():
    # MIN over a list returns the list: ArrowType LIST (tag 25) of a nullable int32 item
    list_type = P.f_bytes(25, P.f_bytes(1, P.field("item", pa.int32())))
    node = (P.f_bytes(1, P.f_str(1, "m") + P.f_bytes(2, list_type) + P.f_varint(3, 1)) + P.f_bytes(1000, list_type) + P.f_varint(2, 1)
            + P.f_varint(4, P.AGG_FN["MIN"]) + P.f_bytes(5, P.col("i")))
    msg = _error([node])
    assert "window MIN" in msg and "list" in msg


def test_functions_outside_the_path_stay_rejected():
    for fn in ("FIRST", "FIRST_IGNORES_NULL"):
        if fn not in P.AGG_FN:
            continue
        assert "not native" in _error([P.window_expr("w", pa.int64(), fn, [P.col("i")])]).lower()
