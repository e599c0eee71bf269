"""ParquetScanExec over files with nested columns: flat columns beside nested siblings (which the JVM side sends as NullType), and
one-level LIST columns read as list columns on the device, value by value against list_scan_reference.py (pq.read_table + the
adapter's element casts).  Floats compare by bits, NaN matches NaN."""
import decimal
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import list_scan_reference as LR
import parquet_nested_pages as NP
from auron_b200 import proto as P
from auron_b200 import runtime
from helpers import run

pytestmark = pytest.mark.gpu

I32, I64, U = pa.int32(), pa.int64(), pa.string()
TS = pa.timestamp


def _scan(paths, schema, proj=None):
    files = [(p, os.path.getsize(p)) for p in (paths if isinstance(paths, list) else [paths])]
    return P.parquet_scan(schema, files, list(range(len(schema))) if proj is None else proj)


def _check(paths, schema, proj=None):
    got = run(_scan(paths, schema, proj), {})
    names = [schema.field(i).name for i in (range(len(schema)) if proj is None else proj)]
    want = {}
    for p in (paths if isinstance(paths, list) else [paths]):
        for k, v in LR.read(p, pa.schema([schema.field(n) for n in names])).items():
            want.setdefault(k, []).extend(v)
    assert got.num_rows == len(want[names[0]])
    for n in names:
        g = LR.canon_column(got[n])
        bad = [i for i, (a, b) in enumerate(zip(g, want[n])) if a != b]
        assert not bad, (n, [(i, g[i], want[n][i]) for i in bad[:5]])
    return got


def _nested_siblings(n, rng):
    ids = np.arange(n)
    return pa.table({
        "l": pa.array([[int(i)] * int(i % 3) if i % 5 else None for i in ids], pa.list_(I64)),
        "a": pa.array(rng.integers(-1000, 1000, n).astype(np.int32), mask=rng.random(n) < 0.1),
        "s": pa.array([{"x": int(i)} if i % 3 else None for i in ids], pa.struct([("x", I32)])),
        "m": pa.array([[("k", int(i))] if i % 4 else None for i in ids], pa.map_(U, I32)),
        "ll": pa.array([[[int(i)], []] if i % 2 else None for i in ids], pa.list_(pa.list_(I32))),
        "ls": pa.array([[{"p": int(i)}] for i in ids], pa.list_(pa.struct([("p", I32)]))),
        "b": pa.array([f"v{int(i) % 97}" for i in ids], mask=rng.random(n) < 0.05),
        "z": pa.array(ids.astype(np.int64)),
    })


@pytest.mark.parametrize("version,codec", [("1.0", "SNAPPY"), ("2.0", "ZSTD"), ("1.0", "NONE")])
def test_flat_columns_beside_nested_siblings(tmp_path, version, codec):
    t = _nested_siblings(20_000, np.random.default_rng(1))
    path = str(tmp_path / "n.parquet")
    pq.write_table(t, path, data_page_version=version, compression=codec, row_group_size=7000)
    # every field the query does not read comes as NullType, as NativeFileSourceScanBase sends it
    sch = pa.schema([pa.field(f.name, f.type if f.name in ("a", "b", "z") else pa.null()) for f in t.schema])
    got = run(_scan(path, sch), {})
    for f in t.schema:
        if f.name in ("a", "b", "z"):
            assert LR.canon_column(got[f.name]) == LR.read(path, pa.schema([f]))[f.name]
        else:
            assert got[f.name].null_count == t.num_rows
    # the same file with only the flat columns in the projection, and with the list read too
    _check(path, pa.schema([("z", I64), ("b", U), ("a", I64)]))
    _check(path, pa.schema([("b", U), ("l", pa.list_(I64)), ("z", I64)]))


def test_fused_path_with_nested_siblings(tmp_path):
    rng = np.random.default_rng(2)
    m = 120_000
    pt = pa.table({"tags": pa.array([["x"] * int(k) for k in rng.integers(0, 3, m)], pa.list_(U)),
                   "item": pa.array(rng.integers(1, 3000, m).astype(np.int32)),
                   "addr": pa.array([{"zip": int(k)} for k in rng.integers(0, 9, m)], pa.struct([("zip", I32)])),
                   "qty": pa.array(rng.integers(1, 101, m).astype(np.int32), mask=rng.random(m) < 0.03),
                   "date": pa.array(rng.integers(2450816, 2452642, m).astype(np.int32), mask=rng.random(m) < 0.04)})
    path = str(tmp_path / "f.parquet")
    pq.write_table(pt, path, compression="SNAPPY", row_group_size=25_000)
    sch = pa.schema([("tags", pa.null()), ("item", I32), ("addr", pa.null()), ("qty", I32), ("date", I32)])
    scan = P.parquet_scan(sch, [(path, os.path.getsize(path))], [1, 3, 4])
    flt = P.filter_(scan, [P.binary("GtEq", P.col("date"), P.lit(2451000, I32)), P.binary("Lt", P.col("date"), P.lit(2452000, I32))])
    plan = P.agg(flt, [P.try_cast(P.col("item"), I64)], ["item"], [P.agg_expr("SUM", [P.col("qty")], I64), P.agg_expr("COUNT", [P.col("qty")], I64)],
                 ["s", "c"], ["PARTIAL", "PARTIAL"])
    with runtime.Task(P.task_definition(plan)) as task:
        out = pa.Table.from_batches(list(task), schema=task.schema)
        fused = sum(v for _, _, name, v in task.metrics() if name == "fused_batches")
    assert fused > 0
    d = pt["date"].to_numpy(zero_copy_only=False)
    keep = ~np.isnan(d.astype(float)) & (np.nan_to_num(d.astype(float)) >= 2451000) & (np.nan_to_num(d.astype(float)) < 2452000)
    exp = {}
    for it, q, k in zip(pt["item"].to_pylist(), pt["qty"].to_pylist(), keep):
        if k:
            s, c = exp.get(it, (None, 0))
            exp[it] = ((s or 0) + q if q is not None else s, c + (q is not None))
    got = {k: (s, c) for k, s, c in zip(*[c.to_pylist() for c in out.columns])}
    assert got == exp


def _dec(unscaled, scale):
    with decimal.localcontext() as c:
        c.prec = 80
        return decimal.Decimal(unscaled).scaleb(-scale)


def _lists(vals, n, rng, null_lists, null_elems):
    out = []
    for i in range(n):
        if null_lists and i % 13 == 5:
            out.append(None)
            continue
        k = int(rng.integers(0, 6)) if i % 17 else 0
        row = [vals[(i + j) % len(vals)] for j in range(k)]
        if null_elems:
            row = [None if (i + j) % 7 == 3 else v for j, v in enumerate(row)]
        out.append(row)
    return out


ELEM = {
    "i8": (pa.int8(), [-128, 127, 0, 1, -1], [pa.int16(), pa.int64()]),
    "i16": (pa.int16(), [-2**15, 2**15 - 1, 0, -1], [pa.int32()]),
    "i32": (I32, [-2**31, 2**31 - 1, 0, 1, -1], [I64, pa.float64(), pa.decimal128(12, 0)]),
    "i64": (I64, [-2**63, 2**63 - 1, 0, -1], [pa.decimal128(20, 0)]),
    "u8": (pa.uint8(), [0, 255, 128], [pa.int16()]),
    "u16": (pa.uint16(), [0, 2**16 - 1, 2**15], [pa.int32()]),
    "u32": (pa.uint32(), [0, 2**32 - 1, 2**31], [pa.int64()]),
    "f32": (pa.float32(), [float("nan"), -0.0, float("inf"), -float("inf"), 1.401298464324817e-45, 3.4028234663852886e38], [pa.float64()]),
    "f64": (pa.float64(), [float("nan"), -0.0, 5e-324, 1.7976931348623157e308, -float("inf")], []),
    "ts_s": (TS("s"), [-1, 0, 2**40], [TS("us")]),
    "ts_ms": (TS("ms"), [-1, 0, 1, -1001, (2**63 - 1) // 1000, (2**63 - 1) // 1000 + 1], [TS("us"), TS("ns"), TS("s")]),
    "ts_us": (TS("us"), [-1, 0, 2**63 - 1, -2**63 + 1], [TS("ms")]),
    "ts_ns": (TS("ns"), [-1, -999_999, 2**63 - 1], [TS("us")]),
    "dt": (pa.date32(), [-2**31, 2**31 - 1, 0, -719162], [I64]),
    "s": (U, ["", "a", "é", "😀", "x" * 5000], [pa.binary()]),
    "b": (pa.binary(), [b"", b"\x00\xff", b"y" * 3000], []),
    "bool": (pa.bool_(), [True, False], []),
    "d9": (pa.decimal128(9, 2), [10**9 - 1, -(10**9 - 1), 0, 1], [pa.decimal128(14, 4)]),
    "d18": (pa.decimal128(18, 3), [10**18 - 1, -(10**18 - 1), 0], [pa.decimal128(21, 6)]),
    "d38": (pa.decimal128(38, 10), [10**38 - 1, -(10**38 - 1), 0], []),
}


def _elem_table(n, rng, null_lists, null_elems, names=ELEM):
    cols = {}
    for name, (t, vals, _) in ELEM.items():
        if name not in names:
            continue
        rows = _lists(vals, n, rng, null_lists, null_elems)
        if pa.types.is_timestamp(t) or pa.types.is_date32(t):
            arr = pa.array(rows, pa.list_(I64 if pa.types.is_timestamp(t) else I32)).cast(pa.list_(t))
        elif pa.types.is_decimal(t):
            arr = pa.array([None if r is None else [None if x is None else _dec(x, t.scale) for x in r] for r in rows], pa.list_(t))
        else:
            arr = pa.array(rows, pa.list_(t))
        cols[name] = arr.cast(pa.list_(pa.field("element", t, nullable=null_elems)))
    fields = [pa.field(k, pa.list_(pa.field("element", v.type.value_type, nullable=null_elems)), nullable=null_lists) for k, v in cols.items()]
    return pa.table(list(cols.values()), schema=pa.schema(fields))


def _read_schemas(t):
    own = {pa.uint8(): pa.int16(), pa.uint16(): pa.int32(), pa.uint32(): pa.int64()}
    base = pa.schema([pa.field(f.name, pa.list_(own.get(f.type.value_type, f.type.value_type))) for f in t.schema])
    out = [base]
    for k in range(3):
        wide = [pa.field(f.name, pa.list_(ELEM[f.name][2][k])) for f in t.schema if len(ELEM[f.name][2]) > k]
        if wide:
            out.append(pa.schema(wide))
    return out


LAYOUTS = [  # (use_dictionary, data page version, compression, null lists, null elements)
    (True, "1.0", "NONE", True, True),
    (False, "2.0", "SNAPPY", True, True),
    (True, "2.0", "ZSTD", False, False),
    (False, "1.0", "LZ4_RAW", False, True),
    (True, "1.0", "SNAPPY", True, False),
]


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: "-".join(str(x) for x in l))
def test_list_of_every_element_type_at_its_edges(tmp_path, layout):
    dict_, page_version, codec, null_lists, null_elems = layout
    t = _elem_table(3000, np.random.default_rng(3), null_lists, null_elems)
    path = str(tmp_path / "e.parquet")
    pq.write_table(t, path, use_dictionary=dict_, data_page_version=page_version, compression=codec, row_group_size=1100, data_page_size=4096,
                   store_decimal_as_integer=True)
    for sch in _read_schemas(t):
        _check(path, sch)
    # decimals on FIXED_LEN_BYTE_ARRAY
    flba = str(tmp_path / "flba.parquet")
    pq.write_table(t.select(["d9", "d18", "d38"]), flba, use_dictionary=dict_, data_page_version=page_version, compression=codec)
    _check(flba, pa.schema([("d9", pa.list_(pa.decimal128(9, 2))), ("d18", pa.list_(pa.decimal128(21, 6))), ("d38", pa.list_(pa.decimal128(38, 10)))]))


@pytest.mark.parametrize("page_version", ["1.0", "2.0"])
@pytest.mark.parametrize("codec", ["NONE", "SNAPPY", "ZSTD", "LZ4_RAW"])
@pytest.mark.parametrize("dict_", [True, False])
@pytest.mark.parametrize("host_snappy", [False, True])
def test_codecs_page_versions_and_dictionaries(tmp_path, monkeypatch, page_version, codec, dict_, host_snappy):
    if host_snappy and codec != "SNAPPY":
        pytest.skip("AURON_HOST_SNAPPY only moves SNAPPY pages")
    if host_snappy:
        monkeypatch.setenv("AURON_HOST_SNAPPY", "1")
    rng = np.random.default_rng(4)
    n = 40_000
    t = pa.table({"id": pa.array(np.arange(n, dtype=np.int64)),
                  "l": pa.array(_lists(list(range(-50, 50)), n, rng, True, True), pa.list_(I64)),
                  "s": pa.array(_lists([f"w{i}" for i in range(30)], n, rng, True, True), pa.list_(U))})
    path = str(tmp_path / "c.parquet")
    pq.write_table(t, path, use_dictionary=dict_, data_page_version=page_version, compression=codec, row_group_size=15_000, data_page_size=8192)
    _check(path, pa.schema([("l", pa.list_(I64)), ("id", I64), ("s", pa.list_(U))]))


def test_many_pages_row_groups_files_and_small_batches(tmp_path, monkeypatch):
    monkeypatch.setenv("AURON_GPU_CHUNK_ROWS", "5000")
    rng = np.random.default_rng(5)
    paths = []
    for k in range(3):
        n = 12_000 + 1000 * k
        t = pa.table({"l": pa.array([[int(x) for x in rng.integers(-9, 9, int(rng.integers(0, 40)))] if rng.random() > 0.1 else None for _ in range(n)],
                                    pa.list_(I32)),
                      "s": pa.array([[f"t{int(x)}" for x in rng.integers(0, 50, int(rng.integers(0, 4)))] for _ in range(n)], pa.list_(U))})
        p = str(tmp_path / f"m{k}.parquet")
        pq.write_table(t, p, compression="SNAPPY", row_group_size=2500 + 500 * k, data_page_size=512, data_page_version=["1.0", "2.0", "1.0"][k])
        paths.append(p)
    _check(paths, pa.schema([("l", pa.list_(I64)), ("s", pa.list_(U))]))


@pytest.mark.parametrize("form", [f for f in NP.FORMS if NP.FORMS[f][1]])
@pytest.mark.parametrize("v2", [False, True])
def test_hand_built_legacy_forms_and_straddling_pages(tmp_path, form, v2):
    rng = np.random.default_rng(6)
    elem_required = form in ("two_level_primitive", "bare_repeated")
    may_be_null = form not in ("two_level_primitive", "bare_repeated", "required_standard")
    rows = []
    for i in range(3000):
        if may_be_null and i % 11 == 0:
            rows.append(None)
            continue
        r = [int(x) for x in rng.integers(-2**31, 2**31, int(rng.integers(0, 9)))]
        rows.append(r if elem_required else [None if j % 4 == 1 else v for j, v in enumerate(r)])
    n_slots = len(NP.slots_of(rows, *NP.levels_of(form, elem_required)))
    cuts = sorted(set(int(c) for c in rng.integers(1, n_slots, 40)))   # most pages start inside a row
    path = str(tmp_path / "h.parquet")
    NP.write(path, form, rows, cuts=cuts, elem_required=elem_required, v2=v2)
    got = _check(path, pa.schema([("l", pa.list_(I64))]))
    assert got["l"].to_pylist() == rows


@pytest.mark.parametrize("form", [f for f in NP.FORMS if not NP.FORMS[f][1]])
def test_unread_shapes_cost_nothing_and_fail_when_projected(tmp_path, form):
    path = str(tmp_path / "u.parquet")
    NP.write(path, form, [])
    assert run(_scan(path, pa.schema([("l", pa.null())])), {}).num_rows == 0
    with pytest.raises(Exception, match=f"cannot read parquet column l \\(a {NP.SHAPES[form]}\\)"):
        run(_scan(path, pa.schema([("l", pa.list_(I32))])), {})


def test_shape_mismatches_name_the_column(tmp_path):
    t = pa.table({"l": pa.array([[1], None], pa.list_(I32)), "x": pa.array([1, 2], I32),
                  "st": pa.array([{"a": 1}, None], pa.struct([("a", I32)]))})
    path = str(tmp_path / "r.parquet")
    pq.write_table(t, path)
    with pytest.raises(Exception, match="cannot read parquet column l \\(a list of physical type 1\\) as int32"):
        run(_scan(path, pa.schema([("l", I32)])), {})
    with pytest.raises(Exception, match="cannot read parquet column x \\(a primitive column, physical type 1\\) as list"):
        run(_scan(path, pa.schema([("x", pa.list_(I32))])), {})
    with pytest.raises(Exception, match="cannot read parquet column st \\(a struct\\)"):
        run(_scan(path, pa.schema([("st", I32)])), {})
    with pytest.raises(Exception, match="cannot read parquet column l.list.element"):
        run(_scan(path, pa.schema([("l", pa.list_(U))])), {})


def test_tags_explode_count_end_to_end(tmp_path):
    rng = np.random.default_rng(7)
    words = ["alpha", "beta", "gamma", "é", "", "delta"]
    n = 150_000
    tags = [None if rng.random() < 0.03 else [None if rng.random() < 0.05 else words[int(x)] for x in rng.integers(0, 6, int(rng.integers(0, 6)))]
            for _ in range(n)]
    tab = pa.table({"id": pa.array(range(n), I64), "tags": pa.array(tags, pa.list_(U))})
    path = str(tmp_path / "tags.parquet")
    pq.write_table(tab, path, compression="SNAPPY", row_group_size=40_000)
    scan = P.parquet_scan(tab.schema, [(path, os.path.getsize(path))], [0, 1])
    gen = P.generate(scan, "Explode", P.col("tags"), [], [("w", U, True)])
    partial = P.agg(gen, [P.col("w")], ["w"], [P.agg_expr("COUNT", [P.col("w")], I64)], ["c"], ["PARTIAL"])
    final = P.agg(partial, [P.col("w")], ["w"], [P.agg_expr("COUNT", [P.lit(None, pa.null())], I64)], ["c"], ["FINAL"])
    got = dict(zip(*[c.to_pylist() for c in run(final, {}).columns]))
    exp = {}
    for r in tags:
        for w in r or []:
            exp[w] = exp.get(w, 0) + (w is not None)
    assert got == exp


def test_list_through_filter_and_project_keeps_the_plan_field(tmp_path):
    n = 30_000
    tab = pa.table({"id": pa.array(range(n), I64), "tags": pa.array([[f"t{i % 7}"] * (i % 4) if i % 9 else None for i in range(n)], pa.list_(U))})
    path = str(tmp_path / "fp.parquet")
    pq.write_table(tab, path, data_page_version="2.0", compression="SNAPPY", row_group_size=9000)
    LT = pa.list_(pa.field("tag", U, nullable=True))
    scan = P.parquet_scan(pa.schema([("id", I64), ("tags", LT)]), [(path, os.path.getsize(path))], [0, 1])
    flt = P.filter_(scan, [P.binary("Gt", P.binary("Modulo", P.col("id"), P.lit(3, I64)), P.lit(0, I64))])
    got = run(P.projection(flt, [P.col("tags"), P.col("id")], ["t", "id"], [LT, I64]), {})
    assert got.schema.field("t").type == LT
    keep = [i for i in range(n) if i % 3 > 0]
    assert got["id"].to_pylist() == keep
    assert got["t"].to_pylist() == [tab["tags"][i].as_py() for i in keep]


def test_a_file_without_the_list_column_reads_null_lists(tmp_path):
    # files written before the array column was added to the table: every row of them is a NULL list, through explode and export
    rng = np.random.default_rng(8)
    with_tags = pa.table({"id": pa.array(range(5000), I64), "tags": pa.array([[f"t{i % 5}"] * (i % 3) if i % 7 else None for i in range(5000)], pa.list_(U))})
    without = pa.table({"id": pa.array(range(5000, 9000), I64)})
    p1, p2, p3 = (str(tmp_path / f"{k}.parquet") for k in ("old", "new", "old2"))
    pq.write_table(without, p1, row_group_size=1500)
    pq.write_table(with_tags, p2, compression="SNAPPY", row_group_size=2000)
    pq.write_table(without.slice(0, int(rng.integers(1, 900))), p3)
    sch = pa.schema([("id", I64), ("tags", pa.list_(U))])
    files = [p1, p2, p3]
    got = run(_scan(files, sch), {})
    want = [None] * without.num_rows + with_tags["tags"].to_pylist() + [None] * pq.read_metadata(p3).num_rows
    assert got["tags"].to_pylist() == want and got["tags"].null_count == want.count(None)
    assert got.schema.field("tags").type == pa.list_(U)
    gen = P.generate(_scan(files, sch), "PosExplode", P.col("tags"), ["id"], [("pos", I32, True), ("w", U, True)], outer=True)
    rows = sorted(zip(*[c.to_pylist() for c in run(gen, {}).columns]), key=lambda r: (r[0], -1 if r[1] is None else r[1]))
    exp = []
    for i, tg in zip(got["id"].to_pylist(), want):
        exp += [(i, k, w) for k, w in enumerate(tg)] if tg else [(i, None, None)]
    assert rows == sorted(exp, key=lambda r: (r[0], -1 if r[1] is None else r[1]))


def test_field_positions_differ_between_files_of_one_batch(tmp_path):
    # b is column chunk 2 in both files, but top-level field 1 in the first (after a struct) and field 2 in the second: each row
    # group must read b's own chunk, never the chunk at b's position in another file
    n = 3000
    a = pa.table({"s": pa.array([{"x": -i, "y": -2 * i} for i in range(n)], pa.struct([("x", I32), ("y", I32)])), "b": pa.array(range(n), I32)})
    b = pa.table({"x": pa.array([-7] * n, I32), "y": pa.array([-9] * n, I32), "b": pa.array(range(n, 2 * n), I32)})
    pa_, pb = str(tmp_path / "a.parquet"), str(tmp_path / "b.parquet")
    pq.write_table(a, pa_, row_group_size=1000)
    pq.write_table(b, pb, row_group_size=1000)
    got = run(_scan([pa_, pb, pa_], pa.schema([("b", I32)])), {})
    assert got["b"].to_pylist() == list(range(n)) + list(range(n, 2 * n)) + list(range(n))
    got = run(_scan([pb, pa_], pa.schema([("y", I32), ("b", I64), ("s", pa.null())])), {})
    assert got["b"].to_pylist() == list(range(n, 2 * n)) + list(range(n))
    assert got["y"].to_pylist() == [-9] * n + [None] * n


@pytest.mark.parametrize("page_version", ["1.0", "2.0"])
@pytest.mark.parametrize("codec", ["NONE", "SNAPPY"])
def test_delta_encoded_list_pages(tmp_path, page_version, codec):
    rng = np.random.default_rng(9)
    n = 20_000
    t = pa.table({"i": pa.array(_lists(list(range(-2**31, -2**31 + 40)) + [2**31 - 1], n, rng, True, True), pa.list_(I32)),
                  "l": pa.array(_lists([-2**63, 2**63 - 1, 0, 5, -5], n, rng, True, True), pa.list_(I64)),
                  "s": pa.array(_lists([f"w{i}" for i in range(50)] + [""], n, rng, True, True), pa.list_(U)),
                  "d": pa.array(_lists(sorted(f"key-{i:05d}" for i in range(300)), n, rng, False, True), pa.list_(U))})
    path = str(tmp_path / "delta.parquet")
    enc = {"i.list.element": "DELTA_BINARY_PACKED", "l.list.element": "DELTA_BINARY_PACKED", "s.list.element": "DELTA_LENGTH_BYTE_ARRAY",
           "d.list.element": "DELTA_BYTE_ARRAY"}
    pq.write_table(t, path, use_dictionary=False, column_encoding=enc, data_page_version=page_version, compression=codec, row_group_size=7000,
                   data_page_size=4096)
    md = pq.ParquetFile(path).metadata.row_group(0)
    assert {e for c in range(4) for e in md.column(c).encodings} >= {"DELTA_BINARY_PACKED", "DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY"}
    _check(path, pa.schema([("i", pa.list_(I64)), ("l", pa.list_(I64)), ("s", pa.list_(U)), ("d", pa.list_(pa.binary()))]))
