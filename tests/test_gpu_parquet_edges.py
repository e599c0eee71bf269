"""ParquetScanExec at the edges of every physical and logical type, page layout and conversion, value by value against the
plain-Python reference (scan_reference.py: pq.read_table + AuronSchemaAdapter's rules).  NaN matches NaN; every other value
matches bit for bit."""
import decimal
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_pages
import scan_reference as R
from auron_b200 import proto as P
from auron_b200 import runtime
from helpers import run

pytestmark = pytest.mark.gpu

I32_MIN, I32_MAX, I64_MIN, I64_MAX = -2**31, 2**31 - 1, -2**63, 2**63 - 1
TS = pa.timestamp


def _scan(path, schema, prune=None):
    return run(P.parquet_scan(schema, [(path, os.path.getsize(path))], list(range(len(schema))), pruning_predicates=prune), {})


def _check(path, schema):
    got = _scan(path, schema)
    want = R.read(path, schema)
    assert got.num_rows == len(next(iter(want.values())))
    for f in schema:
        g = R.canon_array(got[f.name])
        w = want[f.name]
        bad = [i for i, (a, b) in enumerate(zip(g, w)) if a != b]
        assert not bad, (f.name, f.type, [(i, g[i], w[i]) for i in bad[:5]])


def _tile(vals, n, nulls):
    out = [vals[i % len(vals)] for i in range(n)]
    if nulls == "alternating":
        out = [None if i % 2 else v for i, v in enumerate(out)]
    elif nulls == "all":
        out = [None] * n
    return out


DEC_P = [1, 2, 9, 10, 18, 19, 38]
MS_EDGE = I64_MAX // 1000


def _edge_table(n, nulls):
    cols = {
        "i8": (pa.int8(), [-128, 127, 0, 1, -1]),
        "i16": (pa.int16(), [-2**15, 2**15 - 1, 0, 1, -1]),
        "i32": (pa.int32(), [I32_MIN, I32_MAX, 0, 1, -1, 2**24 + 1, -(2**24 + 1)]),
        "i64": (pa.int64(), [I64_MIN, I64_MAX, 0, 1, -1]),
        "u8": (pa.uint8(), [0, 1, 127, 128, 255]),
        "u16": (pa.uint16(), [0, 1, 2**15 - 1, 2**15, 2**16 - 1]),
        "u32": (pa.uint32(), [0, 1, 2**31 - 1, 2**31, 2**32 - 1]),
        "f32": (pa.float32(), [float("nan"), -float("nan"), 0.0, -0.0, float("inf"), -float("inf"), 1.401298464324817e-45, 3.4028234663852886e38]),
        "f64": (pa.float64(), [float("nan"), -float("nan"), 0.0, -0.0, float("inf"), -float("inf"), 5e-324, 1.7976931348623157e308]),
        "ts_s": (TS("s"), [-1, 0, 1, -86401, 2**40]),
        "ts_ms": (TS("ms"), [-1, 0, 1, -1001, MS_EDGE, MS_EDGE + 1, -MS_EDGE, -MS_EDGE - 1]),
        "ts_us": (TS("us"), [-1, 0, 1, -1001, I64_MAX, I64_MIN + 1]),
        "ts_ns": (TS("ns"), [-1, 0, 1, -1001, -999_999, I64_MAX, I64_MIN + 1]),
        "dt": (pa.date32(), [I32_MIN, I32_MAX, 0, -1, -719162, 2932896]),
        "s": (pa.string(), ["", "a", "é", "天", "😀", "a\x00b", "x" * 70_000]),
        "b": (pa.binary(), [b"", b"\x00", b"\x00\x00\xff", b"y" * 66_000]),
    }
    for p in DEC_P:
        m = 10**p - 1
        cols[f"d{p}"] = (pa.decimal128(p, p // 2), [m, -m, 0, 1, -1])
    arrays = {}
    for name, (t, vals) in cols.items():
        v = _tile(vals, n, nulls)
        if pa.types.is_timestamp(t) or pa.types.is_date32(t):
            arrays[name] = pa.array(v, pa.int64() if pa.types.is_timestamp(t) else pa.int32()).cast(t)
        elif pa.types.is_decimal(t):
            arrays[name] = pa.array([None if x is None else _dec(x, t.scale) for x in v], t)
        else:
            arrays[name] = pa.array(v, t)
    return pa.table(arrays)


def _dec(unscaled, scale):
    with decimal.localcontext() as c:
        c.prec = 80
        return decimal.Decimal(unscaled).scaleb(-scale)


def _read_schemas(file_schema):
    """every column at its own type, then at each wider type the conversion table allows"""
    own = pa.schema([pa.field(f.name, {pa.uint8(): pa.int16(), pa.uint16(): pa.int32(), pa.uint32(): pa.int64()}.get(f.type, f.type)) for f in file_schema])
    wide = {"i8": pa.int16(), "i16": pa.int32(), "i32": pa.float64(), "u8": pa.int64(), "u16": pa.int64(), "f32": pa.float64(),
            "ts_s": TS("us"), "ts_ms": TS("us"), "ts_us": TS("ms"), "ts_ns": TS("us"), "dt": pa.int64(), "s": pa.binary()}
    for p in DEC_P:
        if p < 38:
            wide[f"d{p}"] = pa.decimal128(min(38, p + 3), p // 2 + 2)
    alt = pa.schema([pa.field(f.name, wide.get(f.name, own.field(f.name).type)) for f in file_schema if f.name in wide])
    ns_ms = pa.schema([f for f in [pa.field("ts_ns", TS("ms")), pa.field("ts_ms", TS("ns")), pa.field("ts_us", TS("s")), pa.field("i32", pa.int64()),
                                   pa.field("i8", pa.int32())] if f.name in file_schema.names])
    return [own, alt, ns_ms]


LAYOUTS = [  # (use_dictionary, format version, data page version, compression, required, nulls)
    (True, "2.6", "1.0", "NONE", False, "alternating"),
    (False, "2.6", "2.0", "SNAPPY", False, "none"),
    (True, "1.0", "2.0", "ZSTD", True, "none"),
    (False, "2.6", "1.0", "LZ4_RAW", True, "none"),
    (True, "2.6", "2.0", "SNAPPY", False, "all"),
]


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: "-".join(str(x) for x in l))
def test_types_at_their_edges(tmp_path, layout):
    dict_, version, page_version, codec, required, nulls = layout
    t = _edge_table(2100, nulls)
    if version == "1.0":
        t = t.drop_columns(["ts_ns"])      # (format 1.0 has no nanosecond unit: the writer would truncate to microseconds)
    if required:
        t = t.cast(pa.schema([pa.field(f.name, f.type, nullable=False) for f in t.schema]))
    path = str(tmp_path / "edges.parquet")
    pq.write_table(t, path, use_dictionary=dict_, version=version, data_page_version=page_version, compression=codec, row_group_size=1025,
                   data_page_size=2048, write_batch_size=64, store_decimal_as_integer=(codec == "ZSTD"), allow_truncated_timestamps=True,
                   coerce_timestamps=None)
    for schema in _read_schemas(t.schema):
        _check(path, schema)


@pytest.mark.parametrize("chunk_rows", [None, "1000", "1025"])
@pytest.mark.parametrize("rg", [1, 31, 1025])
def test_null_runs_around_words_and_tiles(tmp_path, monkeypatch, chunk_rows, rg):
    # NULL runs that start and end one row either side of multiples of 32 and 1024, row groups of 1, 31 and 1025 rows
    n = 3100
    valid = np.ones(n, bool)
    for b in (32, 64, 1024, 2048):
        valid[b - 1:b + 1] = False
    valid[1023 - 33:1023 + 2] = False
    valid[2500:2600:2] = False
    vals = np.arange(n, dtype=np.int64) * 2654435761 % 2**32 - 2**31
    t = pa.table({"k": pa.array(vals.astype(np.int32), mask=~valid), "ms": pa.array(vals * 10**9, TS("ms"), mask=~valid),
                  "u": pa.array((vals % 2**32).astype(np.uint32), mask=~valid), "d": pa.array(vals, pa.int64(), mask=~valid).cast(pa.decimal128(38, 0)).cast(pa.decimal128(18, 0))})
    path = str(tmp_path / "runs.parquet")
    pq.write_table(t, path, row_group_size=rg, data_page_size=512, write_batch_size=100, compression="SNAPPY")
    if chunk_rows:
        monkeypatch.setenv("AURON_GPU_CHUNK_ROWS", chunk_rows)
    _check(path, pa.schema([("k", pa.int32()), ("ms", TS("us")), ("u", pa.int64()), ("d", pa.decimal128(20, 2))]))


@pytest.mark.parametrize("k", [0, 1, 2, 4, 7, 8, 12, 15, 16, 19, 20])
def test_dictionary_index_widths(tmp_path, k):
    # 2^k and 2^k + 1 entries: index widths 1 .. 21
    for size in (2**k, 2**k + 1):
        n = max(size * 2, 64)
        rng = np.random.default_rng(size)
        vals = (np.arange(n) % size).astype(np.int64) * 7919 - 2**40
        rng.shuffle(vals)
        t = pa.table({"v": pa.array(vals), "w": pa.array(vals.astype(np.int32) if size < 2**16 else (vals % 2**31).astype(np.int32), mask=np.arange(n) % 3 == 0)})
        path = str(tmp_path / f"dict{size}.parquet")
        pq.write_table(t, path, use_dictionary=True, dictionary_pagesize_limit=64 << 20, row_group_size=n, compression="NONE")
        assert pq.ParquetFile(path).metadata.row_group(0).column(0).has_dictionary_page
        _check(path, pa.schema([("v", pa.int64()), ("w", pa.int32())]))


@pytest.mark.parametrize("layout", parquet_pages.layouts(), ids=lambda x: x[0])
@pytest.mark.parametrize("chunk_rows", [None, "1000"])
def test_hand_built_pages(tmp_path, monkeypatch, layout, chunk_rows):
    name, phys, required, pages, dictionary = layout
    path = str(tmp_path / f"{name}.parquet")
    want = parquet_pages.write(path, phys, required, pages, dictionary, stats=True)
    assert pq.read_table(path)["c"].to_pylist() == want
    if chunk_rows:
        monkeypatch.setenv("AURON_GPU_CHUNK_ROWS", chunk_rows)
    t = pa.int32() if phys == "INT32" else pa.int64()
    got = _scan(path, pa.schema([("c", t)]))
    assert got["c"].to_pylist() == want
    if phys == "INT32":   # widened, and as the key of the fused scan -> filter -> aggregate
        assert _scan(path, pa.schema([("c", pa.int64())]))["c"].to_pylist() == want
        _check_agg(path, "c", pa.int32(), None, -2**31, 2**31 - 1)


def _agg_plan(path, key, key_type, lo, hi):
    schema = pa.schema([(key, key_type)])
    scan = P.parquet_scan(schema, [(path, os.path.getsize(path))], [0])
    flt = P.filter_(scan, [P.binary("GtEq", P.col(key), P.lit(lo, key_type)), P.binary("LtEq", P.col(key), P.lit(hi, key_type))])
    return P.agg(flt, [P.try_cast(P.col(key), pa.int64())], ["k"], [P.agg_expr("COUNT", [P.col(key)], pa.int64())], ["c"], ["PARTIAL"])


def _check_agg(path, key, key_type, monkeypatch, lo, hi):
    vals = [v for v in R.read(path, pa.schema([(key, key_type)]))[key]]
    counts = {}
    for v in vals:
        if v is not None and lo <= v <= hi:
            counts[v] = counts.get(v, 0) + 1
    results = []
    for disable in (False, True):
        if disable:
            os.environ["AURON_DISABLE_FUSED_SCAN_AGG"] = "1"
        try:
            with runtime.Task(P.task_definition(_agg_plan(path, key, key_type, lo, hi))) as task:
                got = pa.Table.from_batches(list(task), schema=task.schema)
                fused = sum(v for _, _, name, v in task.metrics() if name == "fused_batches")
        finally:
            os.environ.pop("AURON_DISABLE_FUSED_SCAN_AGG", None)
        assert dict(zip(got.column(0).to_pylist(), got.column(1).to_pylist())) == counts, (path, disable)
        results.append(fused)
    assert results[1] == 0
    return results[0]


def test_fused_aggregate_keys_at_int32_edges_and_uint32(tmp_path):
    rng = np.random.default_rng(4)
    n = 50_000
    lo_keys = (I32_MIN + rng.integers(0, 300, n)).astype(np.int32)
    hi_keys = (I32_MAX - rng.integers(0, 300, n)).astype(np.int32)
    u = (2**31 - 150 + rng.integers(0, 300, n)).astype(np.uint32)      # straddles 2^31: negative if sign-extended
    t = pa.table({"lo": pa.array(lo_keys, mask=rng.random(n) < 0.05), "hi": pa.array(hi_keys), "u": pa.array(u, mask=rng.random(n) < 0.02)})
    path = str(tmp_path / "keys.parquet")
    pq.write_table(t, path, row_group_size=20_000, compression="SNAPPY")
    assert _check_agg(path, "lo", pa.int32(), None, I32_MIN, I32_MIN + 200) > 0
    assert _check_agg(path, "hi", pa.int32(), None, I32_MAX - 200, I32_MAX) > 0
    _check_agg(path, "u", pa.int64(), None, 2**31 - 100, 2**31 + 100)
    _check(path, pa.schema([("u", pa.int64())]))


def _pruned(path, schema, prune, flt):
    scan = P.parquet_scan(schema, [(path, os.path.getsize(path))], list(range(len(schema))), pruning_predicates=prune)
    with runtime.Task(P.task_definition(P.filter_(scan, flt))) as task:
        got = pa.Table.from_batches(list(task), schema=task.schema)
        met = {(op, name): v for _, op, name, v in task.metrics()}
    return got, met.get(("ParquetExec", "row_groups_pruned"), 0)


def test_pruning_uses_converted_statistics(tmp_path):
    n = 40_000
    base = 1_600_000_000_000                                         # milliseconds
    t = pa.table({"ms": pa.array(base + np.arange(n, dtype=np.int64) * 1000, TS("ms")),
                  "u": pa.array((2**31 - 20_000 + np.arange(n)).astype(np.uint32)),
                  "d": pa.array(np.arange(n, dtype=np.int64), pa.int64()).cast(pa.decimal128(38, 2)).cast(pa.decimal128(9, 2))})
    path = str(tmp_path / "prune.parquet")
    pq.write_table(t, path, row_group_size=5_000, store_decimal_as_integer=True)
    # millisecond file read as microseconds: the predicate is in microseconds
    cut = (base + 30_000 * 1000) * 1000
    p = [P.binary("GtEq", P.col("ms"), P.lit(cut, TS("us")))]
    got, pruned = _pruned(path, pa.schema([("ms", TS("us"))]), p, p)
    want = [v for v in R.read(path, pa.schema([("ms", TS("us"))]))["ms"] if v >= cut]
    assert R.canon_array(got["ms"]) == want and len(want) == 10_000
    assert pruned >= 5
    # UINT_32 read as int64: values >= 2^31 are positive
    p = [P.binary("Gt", P.col("u"), P.lit(2**31 + 10_000, pa.int64()))]
    got, pruned = _pruned(path, pa.schema([("u", pa.int64())]), p, p)
    assert got["u"].to_pylist() == [v for v in R.read(path, pa.schema([("u", pa.int64())]))["u"] if v > 2**31 + 10_000]
    assert got.num_rows == 9_999 and pruned >= 5
    # a decimal read at a wider scale: rows are never lost
    sch = pa.schema([("d", pa.decimal128(12, 4))])
    p = [P.binary("GtEq", P.col("d"), P.lit(_dec(35_000_00, 4), pa.decimal128(12, 4)))]
    got, _ = _pruned(path, sch, p, p)
    assert R.canon_array(got["d"]) == [v for v in R.read(path, sch)["d"] if v >= 35_000_00]


REJECT = [  # (file type, table type)
    (pa.int64(), pa.int32()), (pa.int32(), pa.int8()), (pa.int16(), pa.int8()), (pa.int32(), pa.int16()), (pa.uint8(), pa.int8()),
    (pa.uint16(), pa.int16()), (pa.uint32(), pa.int32()), (pa.uint64(), pa.int64()), (pa.uint64(), pa.decimal128(20, 0)),
    (pa.uint32(), pa.float64()), (pa.decimal128(9, 2), pa.decimal128(9, 1)), (pa.decimal128(9, 2), pa.decimal128(9, 3)),
    (pa.decimal128(20, 2), pa.decimal128(20, 1)), (pa.decimal128(9, 2), pa.int64()), (pa.decimal128(9, 2), pa.float64()),
    (pa.float64(), pa.float32()), (pa.int32(), pa.float32()), (pa.string(), pa.int32()), (pa.int32(), pa.string()),
    (pa.date32(), pa.float64()), (TS("ms"), pa.int32()), (pa.float32(), pa.int32()),
]


@pytest.mark.parametrize("src,dst", REJECT, ids=lambda x: str(x))
def test_pairs_outside_the_table_are_rejected(tmp_path, src, dst):
    vals = {pa.string(): ["a"], pa.date32(): [1]}.get(src, [1])
    if pa.types.is_decimal(src):
        vals = [_dec(1, src.scale)]
    path = str(tmp_path / "r.parquet")
    for dec_int in (False, True):
        pq.write_table(pa.table({"col_x": pa.array(vals, src)}), path, store_decimal_as_integer=dec_int)
        with pytest.raises(runtime.AuronError, match="cannot read parquet column col_x"):
            _scan(path, pa.schema([("col_x", dst)]))


def test_byte_stream_split_names_the_encoding(tmp_path):
    path = str(tmp_path / "bss.parquet")
    pq.write_table(pa.table({"f": pa.array([1.5, 2.5], pa.float64())}), path, use_dictionary=False, use_byte_stream_split=["f"])
    with pytest.raises(runtime.AuronError, match="BYTE_STREAM_SPLIT"):
        _scan(path, pa.schema([("f", pa.float64())]))
