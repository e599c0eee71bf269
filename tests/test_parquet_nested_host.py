"""The scan's walk over a nested Parquet schema, on the CPU: auron_b200_parquet_describe prints every leaf with its levels and the
top-level field and shape it belongs to, and counts the rows and values of list pages with the scan's host level walk.  Checked
against pyarrow's own schema for files pyarrow writes, and against the rules of parquet-format's LogicalTypes.md for hand-built
files in every legacy list form.  Also pins list_scan_reference.py, the plain-Python reference of the GPU list tests."""
import ctypes as C
import json

import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import list_scan_reference as LR
import parquet_nested_pages as NP
from auron_b200 import runtime


def _describe(path):
    L = runtime.lib()
    L.auron_b200_parquet_describe.restype = C.c_int64
    L.auron_b200_parquet_describe.argtypes = [C.c_char_p, C.c_char_p, C.c_int64]
    buf = C.create_string_buffer(8 << 20)
    assert L.auron_b200_parquet_describe(path.encode(), buf, len(buf)) > 0, buf.value
    return json.loads(buf.value.decode())


def _nested_table(n):
    rows = range(n)
    return pa.table({
        "a": pa.array([i if i % 7 else None for i in rows], pa.int32()),
        "l": pa.array([None if i % 11 == 0 else [] if i % 5 == 0 else [i, None, -i][: 1 + i % 3] for i in rows], pa.list_(pa.int64())),
        "s": pa.array([{"x": i, "y": str(i)} if i % 3 else None for i in rows], pa.struct([("x", pa.int32()), ("y", pa.string())])),
        "m": pa.array([[("k%d" % i, i)] if i % 4 else None for i in rows], pa.map_(pa.string(), pa.int32())),
        "b": pa.array([str(i) for i in rows]),
        "ll": pa.array([[[i], [], None] if i % 2 else None for i in rows], pa.list_(pa.list_(pa.int32()))),
        "ls": pa.array([[{"p": i}] if i % 2 else [] for i in rows], pa.list_(pa.struct([("p", pa.int16())]))),
        "r": pa.array([[str(i)] * (i % 4) for i in rows], pa.list_(pa.field("item", pa.string(), nullable=False))),
        "z": pa.array(list(rows), pa.int64()),
    }, schema=pa.schema([pa.field("a", pa.int32()), pa.field("l", pa.list_(pa.int64())),
                         pa.field("s", pa.struct([("x", pa.int32()), ("y", pa.string())])), pa.field("m", pa.map_(pa.string(), pa.int32())),
                         pa.field("b", pa.string()), pa.field("ll", pa.list_(pa.list_(pa.int32()))),
                         pa.field("ls", pa.list_(pa.struct([("p", pa.int16())]))),
                         pa.field("r", pa.list_(pa.field("item", pa.string(), nullable=False)), nullable=False), pa.field("z", pa.int64(), nullable=False)]))


SHAPE = {"a": "primitive", "l": "list", "s": "struct", "m": "map", "b": "primitive", "ll": "list of lists", "ls": "list of structs", "r": "list",
         "z": "primitive"}


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("compression", ["NONE", "SNAPPY"])
def test_describe_walks_a_nested_schema(tmp_path, version, compression):
    t = _nested_table(3000)
    path = str(tmp_path / "n.parquet")
    pq.write_table(t, path, data_page_version=version, compression=compression, row_group_size=1200, data_page_size=2048)
    d = _describe(path)
    sch = pq.ParquetFile(path).schema
    assert len(d["leaves"]) == len(sch)
    for i, leaf in enumerate(d["leaves"]):
        ref = sch.column(i)
        assert (leaf["path"], leaf["max_def"], leaf["max_rep"], leaf["chunk"]) == (ref.path, ref.max_definition_level, ref.max_repetition_level, i)
        assert leaf["field"] == ref.path.split(".")[0]
        assert leaf["shape"] == SHAPE[leaf["field"]]
    assert [f["name"] for f in d["fields"]] == t.column_names
    assert [f["shape"] for f in d["fields"]] == [SHAPE[n] for n in t.column_names]
    # flat fields keep the levels of a flat schema; b sits after four nested fields and reads its own chunk
    by = {f["name"]: f for f in d["fields"]}
    assert d["leaves"][by["b"]["leaf"]]["path"] == "b" and d["leaves"][by["z"]["leaf"]]["max_def"] == 0
    assert (by["l"]["list_def"], by["l"]["elem_def"]) == (1, 2) and (by["r"]["list_def"], by["r"]["elem_def"]) == (0, 1)
    for f in d["fields"]:
        assert (f["leaf"] >= 0) == (f["shape"] in ("primitive", "list"))
    # the host level walk: rows (rep == 0) and non-null values (def == max_def) of every page of a repeated leaf
    for g, rg in enumerate(d["row_groups"]):
        rows = pq.ParquetFile(path).metadata.row_group(g).num_rows
        for c, cm in enumerate(rg["columns"]):
            if d["leaves"][c]["max_rep"] == 0:
                assert "level_rows" not in cm
                continue
            assert cm["level_pages"] == cm["data_pages"] and cm["level_rows"] == rows, (c, cm)
        lo = g * 1200
        l_vals = t["l"].slice(lo, rows).combine_chunks().flatten()
        assert rg["columns"][by["l"]["leaf"]]["level_values"] == len(l_vals) - l_vals.null_count


ROWS = [[1, 2, 3], None, [], [None], [4], [5, None, 6, 7, 8, 9, 10, 11, 12], [], None, [2**31 - 1, -2**31]] * 3 + [[i for i in range(40)]]


@pytest.mark.parametrize("form", list(NP.FORMS))
@pytest.mark.parametrize("v2", [False, True])
def test_legacy_list_forms_classify_as_the_rules_say(tmp_path, form, v2):
    path = str(tmp_path / f"{form}.parquet")
    readable = NP.FORMS[form][1]
    elem_required = form in ("two_level_primitive", "bare_repeated")
    rows = ROWS
    if form in ("two_level_primitive", "bare_repeated", "required_standard"):
        rows = [r for r in rows if r is not None]
    if elem_required:
        rows = [[v for v in r if v is not None] for r in rows]
    n_slots = len(NP.slots_of(rows, *NP.levels_of(form, elem_required))) if readable else 0
    cuts = (2, 5, 9, 30, n_slots - 3)   # pages that start inside a row
    NP.write(path, form, rows, cuts=cuts, elem_required=elem_required, v2=v2)
    d = _describe(path)
    (f,) = d["fields"]
    assert f["name"] == "l" and f["shape"] == NP.SHAPES[form]
    if not readable:
        assert f["leaf"] == -1
        return
    list_def, elem_def, max_def = NP.levels_of(form, elem_required)
    leaf = d["leaves"][f["leaf"]]
    assert (f["list_def"], f["elem_def"], leaf["max_def"], leaf["max_rep"]) == (list_def, elem_def, max_def, 1)
    (cm,) = d["row_groups"][0]["columns"]
    assert cm["level_rows"] == len(rows) and cm["data_pages"] == len(cuts) + 1
    assert cm["level_values"] == sum(v is not None for r in rows if r for v in r)
    # an independent reader agrees with the writer: the rows read back
    assert pq.read_table(path)["l"].to_pylist() == rows


def test_list_scan_reference_is_pinned(tmp_path):
    path = str(tmp_path / "r.parquet")
    t = pa.table({"i": pa.array([[1, None, -2**31], None, []], pa.list_(pa.int32())),
                  "ts": pa.array([[0, 1], [None], [-1001]], pa.list_(pa.int64())).cast(pa.list_(pa.timestamp("ms"))),
                  "f": pa.array([[float("nan"), -0.0], [], None], pa.list_(pa.float32())),
                  "s": pa.array([["a", None], None, [""]], pa.list_(pa.string())),
                  "x": pa.array([7, None, 9], pa.int32())})
    pq.write_table(t, path)
    sch = pa.schema([("i", pa.list_(pa.int64())), ("ts", pa.list_(pa.timestamp("us"))), ("f", pa.list_(pa.float64())), ("s", pa.list_(pa.string())),
                     ("x", pa.int64()), ("missing", pa.list_(pa.int32()))])
    got = LR.read(path, sch)
    assert got["i"] == [[1, None, -2**31], None, []]
    assert got["ts"] == [[0, 1000], [None], [-1001000]]
    assert got["f"] == [["nan", 0x8000000000000000], [], None]
    assert got["s"] == [[b"a", None], None, [b""]]
    assert got["x"] == [7, None, 9] and got["missing"] == [None, None, None]
    # the engine's side of the comparison: a sliced list whose offsets do not start at 0
    arr = pa.array([[9], [1, None], None, [3]], pa.list_(pa.int32())).slice(1, 3)
    assert LR.canon_column(arr) == [[1, None], None, [3]]
