"""explode / posexplode, split, array() and list columns on the GPU, against generate_reference.py (the reference's semantics restated
in Python; goldens pinned in test_generate_reference_host.py).  Floats are compared by their bits."""
import datetime as dt
import decimal
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from auron_b200 import proto as P
from auron_b200 import runtime
from generate_reference import explode, make_array, string_split

pytestmark = pytest.mark.gpu

U = pa.string()
I32 = pa.int32()
I64 = pa.int64()
SEPARATORS = [",", ", ", ":", ";", "#", "@", "_", "-", "|", "."]   # ShimsImpl.scala:563-572


def _run(plan, inputs):
    return runtime.run_task(P.task_definition(plan), inputs)


def _key(v):   # floats by bits: NaN payloads and -0.0 are values of their own
    if isinstance(v, float):
        return ("f", struct.pack("<d", v))
    if isinstance(v, list):
        return tuple(_key(x) for x in v)
    return v


def _py(a) -> list:
    """to_pylist, with timestamps as their int64 values (Python's datetime ends at year 9999)"""
    t = a.type
    if pa.types.is_timestamp(t):
        return a.cast(I64).to_pylist()
    if pa.types.is_list(t) and pa.types.is_timestamp(t.value_type):
        return a.cast(pa.list_(I64)).to_pylist()
    return a.to_pylist()


def _rows(t: pa.Table):
    return [tuple(_key(v) for v in r) for r in zip(*[_py(c) for c in t.columns])] if t.num_columns else []


def _f32(vals):
    return [None if v is None else struct.unpack("<f", struct.pack("<f", v))[0] for v in vals]


D38 = pa.decimal128(38, 0)
BIG = decimal.Decimal(10 ** 38 - 1)
NEG_BIG = decimal.Decimal(-(10 ** 38 - 1))   # (unary minus would round to the context's 28 digits)
EDGES = {
    "bool": (pa.bool_(), [True, False, None, True]),
    "int8": (pa.int8(), [-128, 127, 0, None, -1]),
    "int16": (pa.int16(), [-32768, 32767, None, 0]),
    "int32": (I32, [-2 ** 31, 2 ** 31 - 1, 0, None]),
    "int64": (I64, [-2 ** 63, 2 ** 63 - 1, None, 1]),
    "float32": (pa.float32(), _f32([float("nan"), -0.0, 0.0, float("inf"), -float("inf"), 3.4e38, None, 1e-45])),
    "float64": (pa.float64(), [float("nan"), -0.0, 0.0, float("-inf"), 1.7976931348623157e308, None, 5e-324]),
    "date32": (pa.date32(), [dt.date(1, 1, 1), dt.date(9999, 12, 31), None, dt.date(1970, 1, 1)]),
    "date64": (pa.date64(), [dt.date(1, 1, 1), None, dt.date(2024, 2, 29)]),
    "ts_s": (pa.timestamp("s"), [0, -2 ** 40, None, 2 ** 40]),
    "ts_ms": (pa.timestamp("ms"), [0, -2 ** 50, None]),
    "ts_us": (pa.timestamp("us", tz="UTC"), [2 ** 62, None, -2 ** 62]),
    "ts_ns": (pa.timestamp("ns"), [-2 ** 63 + 1, 2 ** 63 - 1, None]),
    "decimal38": (D38, [BIG, NEG_BIG, None, decimal.Decimal(0)]),
    "utf8": (U, ["", "a", "é", "€", "😀x", None, "longer string with spaces"]),
    "binary": (pa.binary(), [b"", b"\x00\xff", None, b"abc"]),
}


def _list_column(t, vals, rng, n_rows=300, sliced=True):
    """lists of 0..5 elements drawn from vals, with NULL lists, as a non-zero-based and sliced Arrow array"""
    lists = []
    for _ in range(n_rows):
        k = int(rng.integers(0, 6))
        lists.append(None if rng.random() < 0.15 else [vals[int(rng.integers(0, len(vals)))] for _ in range(k)])
    pad = [vals[0]] * 3   # elements before the first list: offsets that do not start at 0
    flat = pad + [v for lst in lists for v in (lst or [])]
    offs, o = [], len(pad)
    for lst in lists:
        offs.append(o)
        o += len(lst) if lst else 0
    offs.append(o)
    mask = pa.array([lst is None for lst in lists])
    arr = pa.ListArray.from_arrays(pa.array(offs, I32), pa.array(flat, t), mask=mask)
    if sliced:
        return arr.slice(7, n_rows - 20), lists[7:n_rows - 13]
    return arr, lists


@pytest.mark.parametrize("name", sorted(EDGES))
@pytest.mark.parametrize("func,outer", [("Explode", False), ("Explode", True), ("PosExplode", False), ("PosExplode", True)])
def test_explode_every_element_type(name, func, outer):
    t, vals = EDGES[name]
    rng = np.random.default_rng(len(name) * 7 + outer)
    arr, lists = _list_column(t, vals, rng)
    ids = list(range(len(lists)))
    tab = pa.table({"id": pa.array(ids, I64), "l": arr, "s": pa.array([f"r{i}" if i % 5 else None for i in ids], U)})
    gout = ([("pos", I32, False)] if func == "PosExplode" else []) + [("v", t, True)]
    plan = P.generate(P.ffi_reader(tab.schema, "t"), func, P.col("l"), ["s", "id"], gout, outer)
    got = _run(plan, {"t": tab.to_batches(max_chunksize=97)})
    exp = explode([(s, i) for s, i in zip(tab["s"].to_pylist(), ids)], _py(arr), pos=func == "PosExplode", outer=outer)
    assert _rows(got) == [tuple(_key(v) for v in r) for r in exp]
    assert got.schema.field("v").type == t


@pytest.mark.parametrize("required", [[], ["b"], ["b", "a"]])
def test_explode_several_batches_under_a_filter(required):
    rng = np.random.default_rng(3)
    arr, lists = _list_column(I32, [1, 2, None, -5], rng, n_rows=5000, sliced=False)
    tab = pa.table({"a": pa.array(rng.integers(0, 10, len(lists)), I64), "l": arr, "b": pa.array([f"x{i}" for i in range(len(lists))])})
    flt = P.filter_(P.ffi_reader(tab.schema, "t"), [P.binary("Lt", P.col("a"), P.lit(6, I64))])
    got = _run(P.generate(flt, "Explode", P.col("l"), required, [("v", I32, True)], outer=True), {"t": tab.to_batches(max_chunksize=700)})
    cols = {c: tab[c].to_pylist() for c in ("a", "b")}
    keep = [i for i, a in enumerate(cols["a"]) if a < 6]
    exp = explode([tuple(cols[c][i] for c in required) for i in keep], [lists[i] for i in keep], outer=True)
    assert _rows(got) == exp


def _split_table(rng, n, sep):
    alphabet = ["a", "b", "é", "€", sep, sep, " "]
    vals = []
    for _ in range(n):
        k = int(rng.integers(0, 12))
        vals.append(None if rng.random() < 0.05 else "".join(alphabet[int(x)] for x in rng.integers(0, len(alphabet), k)))
    return pa.table({"s": pa.array(vals, U)})


@pytest.mark.parametrize("sep", SEPARATORS + ["<=>", "--"])
def test_split_fuzz(sep):
    tab = _split_table(np.random.default_rng(ord(sep[0])), 200_000, sep)
    plan = P.projection(P.ffi_reader(tab.schema, "t"), [P.scalar_fn("Spark_StringSplit", [P.col("s"), P.lit(sep, U)], pa.list_(U))], ["p"], [pa.list_(U)])
    got = _run(plan, {"t": tab.to_batches(max_chunksize=60_000)})
    assert got["p"].to_pylist() == [string_split(s, sep) for s in tab["s"].to_pylist()]


def test_split_edges_and_a_computed_argument():
    vals = ["", None, ",", ",a", "a,", ",,", "A,B,,C", "---", "--", "-----"]
    tab = pa.table({"s": pa.array(vals, U)})
    lower = P.scalar_fn("Lower", [P.col("s")], U)
    plan = P.projection(P.ffi_reader(tab.schema, "t"), [P.scalar_fn("Spark_StringSplit", [lower, P.lit(",", U)], pa.list_(U)),
                                                        P.scalar_fn("Spark_StringSplit", [P.col("s"), P.lit("--", U)], pa.list_(U))],
                        ["p", "q"], [pa.list_(U), pa.list_(U)])
    got = _run(plan, {"t": [tab.to_batches()[0]]})
    assert got["p"].to_pylist() == [string_split(None if s is None else s.lower(), ",") for s in vals]
    assert got["q"].to_pylist() == [string_split(s, "--") for s in vals]


def test_split_of_rows_of_many_megabytes():
    rng = np.random.default_rng(5)
    many = ",".join("".join(chr(97 + int(c)) for c in rng.integers(0, 26, int(k))) for k in rng.integers(0, 9, 4_000_000))
    assert len(many) >= 16 << 20
    none = "x" * (16 << 20)
    tab = pa.table({"s": pa.array([many, "a,b", none], U)})
    split = P.scalar_fn("Spark_StringSplit", [P.col("s"), P.lit(",", U)], pa.list_(U))
    got = _run(P.projection(P.ffi_reader(tab.schema, "t"), [split], ["p"], [pa.list_(U)]), {"t": tab.to_batches()})
    assert got["p"].to_pylist() == [string_split(s, ",") for s in tab["s"].to_pylist()]


ARRAY_TYPES = ["bool", "int8", "int32", "int64", "float32", "float64", "date32", "ts_us", "decimal38", "utf8", "binary"]


@pytest.mark.parametrize("name", ARRAY_TYPES)
@pytest.mark.parametrize("k", [1, 12])
def test_make_array_and_list_literals(name, k):
    t, vals = EDGES[name]
    rng = np.random.default_rng(k)
    n = 1000
    cols = {f"c{j}": pa.array([vals[int(x)] for x in rng.integers(0, len(vals), n)], t) for j in range(k)}
    tab = pa.table(cols)
    lit_val = next(v for v in vals if v is not None)
    args = [P.col(f"c{j}") if j % 3 else P.lit(lit_val, t) for j in range(k)]   # literal arguments are broadcast
    lt = pa.list_(t)
    lit_list = [vals[0], None, vals[-1]]
    exprs = [P.scalar_fn("Spark_MakeArray", args, lt), P.lit(lit_list, lt), P.lit(None, lt)]
    got = _run(P.projection(P.ffi_reader(tab.schema, "t"), exprs, ["a", "k", "n"], [lt, lt, lt]), {"t": tab.to_batches(max_chunksize=300)})
    cols_py = [_py(tab[f"c{j}"]) if j % 3 else [lit_val] * n for j in range(k)]
    assert [_key(v) for v in _py(got["a"])] == [_key(v) for v in make_array(*cols_py)]
    assert [_key(v) for v in _py(got["k"])] == [_key(lit_list)] * n
    assert got["n"].to_pylist() == [None] * n


def test_explode_of_a_list_literal():
    tab = pa.table({"id": pa.array(range(50), I64)})
    plan = P.generate(P.ffi_reader(tab.schema, "t"), "PosExplode", P.lit([7, None, 9], pa.list_(I32)), ["id"], [("p", I32, False), ("v", I32, True)])
    got = _run(plan, {"t": tab.to_batches()})
    assert _rows(got) == explode([(i,) for i in range(50)], [[7, None, 9]] * 50, pos=True)


def test_pieces_of_a_small_chunk_with_a_row_longer_than_a_piece(monkeypatch):
    monkeypatch.setenv("AURON_GPU_CHUNK_ROWS", "1000")
    lists = [[i] * (i % 7) for i in range(3000)] + [list(range(4500))] + [None, []]
    tab = pa.table({"id": pa.array(range(len(lists)), I64), "l": pa.array(lists, pa.list_(I64))})
    plan = P.generate(P.ffi_reader(tab.schema, "t"), "PosExplode", P.col("l"), ["id"], [("p", I32, False), ("v", I64, True)], outer=True)
    with runtime.Task(P.task_definition(plan), {"t": tab.to_batches()}) as task:
        parts = list(task)
    assert len(parts) > 10 and max(b.num_rows for b in parts) == 4500
    got = pa.Table.from_batches(parts)
    assert _rows(got) == explode([(i,) for i in range(len(lists))], lists, pos=True, outer=True)


def test_required_strings_beyond_int32_offsets_come_out_in_pieces():
    # 40 rows of a 1 MiB string, each exploded into 60 rows: 2.4 GiB of copies of the string column
    s = ["%02d" % i + "x" * ((1 << 20) - 2) for i in range(40)]
    tab = pa.table({"s": pa.array(s, U), "l": pa.array([list(range(60))] * 40, pa.list_(I32))})
    gen = P.generate(P.ffi_reader(tab.schema, "t"), "Explode", P.col("l"), ["s"], [("v", I32, True)])
    proj = P.projection(gen, [P.scalar_fn("CharacterLength", [P.col("s")], I32), P.scalar_fn("Substr", [P.col("s"), P.lit(1, I64), P.lit(2, I64)], U), P.col("v")],
                        ["n", "k", "v"], [I32, U, I32])
    agg = P.agg(proj, [P.col("k")], ["k"], [P.agg_expr("SUM", [P.col("n")], I64), P.agg_expr("SUM", [P.col("v")], I64), P.agg_expr("COUNT", [P.col("v")], I64)],
                ["n", "v", "c"], ["PARTIAL"] * 3)
    got = sorted(_rows(_run(agg, {"t": tab.to_batches()})))
    assert got == [("%02d" % i, 60 << 20, sum(range(60)), 60) for i in range(40)]


def test_list_columns_pass_through_and_export():
    rng = np.random.default_rng(9)
    arr, _ = _list_column(U, EDGES["utf8"][1], rng, n_rows=2000)
    tab = pa.table({"a": pa.array(range(len(arr)), I64), "l": arr})
    src = P.ffi_reader(tab.schema, "t")
    flt = P.filter_(src, [P.binary("Gt", P.col("a"), P.lit(100, I64))])
    plans = {
        "filter": (flt, tab.filter(pc.greater(tab["a"], 100))),
        "limit": (P.limit(src, 500, 10), tab.slice(10, 490)),
        "union": (P.union([src, P.ffi_reader(tab.schema, "u")], tab.schema), pa.concat_tables([tab, tab])),
        "rename": (P.rename_columns(P.f_bytes(19, P.f_bytes(1, src)), ["x", "y"]), tab),
        "project": (P.projection(flt, [P.col("l")], ["l"], [tab.schema.field("l").type]), tab.filter(pc.greater(tab["a"], 100)).select(["l"])),
    }
    for name, (plan, exp) in plans.items():
        inputs = {"t": tab.to_batches(max_chunksize=333), "u": tab.to_batches(max_chunksize=333)}
        got = _run(plan, inputs)
        assert [c.to_pylist() for c in got.columns] == [c.to_pylist() for c in exp.columns], name
        assert got.schema.types == exp.schema.types, name


def _word_table(rng, n):
    words = ["alpha", "beta", "gamma", "é", "", "delta"]
    vals = [None if rng.random() < 0.03 else ",".join(words[int(x)] for x in rng.integers(0, len(words), int(rng.integers(0, 6)))) for _ in range(n)]
    return pa.table({"id": pa.array(range(n), I64), "tags": pa.array(vals, U)})


@pytest.mark.parametrize("func,outer", [("Explode", False), ("PosExplode", True)])
def test_parquet_split_explode_count_end_to_end(tmp_path, func, outer):
    tab = _word_table(np.random.default_rng(11), 150_000)
    path = str(tmp_path / "tags.parquet")
    pq.write_table(tab, path, compression="SNAPPY", row_group_size=40_000)
    scan = P.parquet_scan(tab.schema, [(path, os.path.getsize(path))], [0, 1])
    LU = pa.list_(U)
    proj = P.projection(scan, [P.col("id"), P.scalar_fn("Spark_StringSplit", [P.col("tags"), P.lit(",", U)], LU)], ["id", "parts"], [I64, LU])
    gout = ([("pos", I32, True)] if func == "PosExplode" else []) + [("w", U, True)]
    gen = P.generate(proj, func, P.col("parts"), [], gout, outer)
    partial = P.agg(gen, [P.col("w")], ["w"], [P.agg_expr("COUNT", [P.col("w")], I64)], ["c"], ["PARTIAL"])
    final = P.agg(partial, [P.col("w")], ["w"], [P.agg_expr("COUNT", [P.lit(None, pa.null())], I64)], ["c"], ["FINAL"])
    got = dict(zip(*[c.to_pylist() for c in _run(final, {}).columns]))
    exp = {}
    for r in explode([()] * tab.num_rows, [string_split(s, ",") for s in tab["tags"].to_pylist()], pos=func == "PosExplode", outer=outer):
        w = r[-1]
        exp[w] = exp.get(w, 0) + (w is not None)
    assert got == exp


def test_split_returned_to_the_host():
    tab = _word_table(np.random.default_rng(12), 20_000)
    LU = pa.list_(pa.field("element", U, nullable=False))
    got = _run(P.projection(P.ffi_reader(tab.schema, "t"), [P.scalar_fn("Spark_StringSplit", [P.col("tags"), P.lit(",", U)], LU)], ["p"], [LU]),
               {"t": tab.to_batches(max_chunksize=5000)})
    assert got.schema.field("p").type == LU   # the child field keeps the plan's name and nullability
    assert got["p"].to_pylist() == [string_split(s, ",") for s in tab["tags"].to_pylist()]
