"""CPU side of the Parquet scan's conversions: the plain-Python reference (scan_reference.py) against hand-computed values,
the engine's metadata reader against pyarrow's view of the logical types, and the hand-built page writer against pyarrow."""
import ctypes as C
import json

import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_pages
import scan_reference as R
from auron_b200 import runtime

I64_MAX = 2**63 - 1
TS = pa.timestamp


@pytest.mark.parametrize("v,src,dst,want", [
    # timestamps: finer unit x 10^3k (NULL past int64), coarser unit truncates toward zero
    (-1, TS("ns"), TS("us"), 0),
    (-999, TS("ns"), TS("us"), 0),
    (-1000, TS("ns"), TS("us"), -1),
    (-1001, TS("ns"), TS("us"), -1),
    (1999, TS("us"), TS("ms"), 1),
    (-1, TS("ms"), TS("s"), 0),
    (I64_MAX // 1000, TS("ms"), TS("us"), I64_MAX // 1000 * 1000),
    (I64_MAX // 1000 + 1, TS("ms"), TS("us"), None),
    (-(I64_MAX // 1000), TS("ms"), TS("us"), -(I64_MAX // 1000) * 1000),
    (-(I64_MAX // 1000) - 1, TS("ms"), TS("us"), None),
    (I64_MAX // 10**6, TS("ms"), TS("ns"), I64_MAX // 10**6 * 10**6),
    (I64_MAX // 10**6 + 1, TS("ms"), TS("ns"), None),
    (5, TS("us"), TS("us"), 5),
    (7, TS("ms"), pa.int64(), 7),
    (7, pa.int64(), TS("us"), 7),
    # integers
    (2**32 - 1, pa.uint32(), pa.int64(), 2**32 - 1),
    (2**31, pa.uint32(), pa.int64(), 2**31),
    (255, pa.uint8(), pa.int16(), 255),
    (2**31, pa.int64(), pa.int32(), None),
    (-2**31, pa.int64(), pa.int32(), -2**31),
    (-2**31, pa.int32(), pa.int64(), -2**31),
    (-2**31, pa.int32(), pa.float64(), 0xC1E0000000000000),
    (2**24 + 1, pa.int32(), pa.float64(), 0x4170000010000000),
    (-5, pa.int32(), pa.decimal128(9, 2), -5),                  # integer -> decimal: value copy
    # decimals: x 10^(s2 - s1), NULL past p2 digits
    (10**7 - 1, pa.decimal128(7, 2), pa.decimal128(9, 4), (10**7 - 1) * 100),
    (-(10**7 - 1), pa.decimal128(7, 2), pa.decimal128(9, 4), -(10**7 - 1) * 100),
    (10**7 - 1, pa.decimal128(7, 2), pa.decimal128(7, 3), None),
    (10**18 - 1, pa.decimal128(18, 0), pa.decimal128(38, 20), (10**18 - 1) * 10**20),
    (-(10**38 - 1), pa.decimal128(38, 10), pa.decimal128(38, 10), -(10**38 - 1)),
    (-(10**9 - 1), pa.decimal128(9, 9), pa.decimal128(19, 19), -(10**9 - 1) * 10**10),
    # floats: bits, every NaN alike
    (float("nan"), pa.float32(), pa.float64(), "nan"),
    (-0.0, pa.float32(), pa.float64(), 0x8000000000000000),
    (1.401298464324817e-45, pa.float32(), pa.float64(), 0x36A0000000000000),
    (None, pa.int32(), pa.int64(), None),
])
def test_reference_rules(v, src, dst, want):
    assert R.convert_value(v, src, dst) == want


def test_reference_overflow_edges_are_exact():
    # the edges above, restated from int64's limits: -2^63 = -9223372036854775808
    assert -(I64_MAX // 1000) - 1 == -9223372036854776
    assert (-9223372036854776) * 1000 < -2**63 and R.convert_value(-9223372036854776, TS("ms"), TS("us")) is None
    assert R.convert_value(-9223372036854775, TS("ms"), TS("us")) == -9223372036854775000


def _describe(path):
    L = runtime.lib()
    L.auron_b200_parquet_describe.restype = C.c_int64
    L.auron_b200_parquet_describe.argtypes = [C.c_char_p, C.c_char_p, C.c_int64]
    buf = C.create_string_buffer(1 << 22)
    assert L.auron_b200_parquet_describe(path.encode(), buf, len(buf)) > 0, buf.value
    return json.loads(buf.value.decode())


_LK = {"NONE": 0, "STRING": 1, "DECIMAL": 2, "DATE": 3, "TIMESTAMP": 4, "INT": 5}
_UNIT = {"milliseconds": 1, "microseconds": 2, "nanoseconds": 3}


@pytest.mark.parametrize("version", ["1.0", "2.6"])
@pytest.mark.parametrize("coerce", [None, "ms"])
@pytest.mark.parametrize("dec_int", [False, True])
def test_describe_reports_logical_types(tmp_path, version, coerce, dec_int):
    t = pa.table({
        "i8": pa.array([-128, 127], pa.int8()), "i16": pa.array([1, 2], pa.int16()), "i32": pa.array([1, 2], pa.int32()), "i64": pa.array([1, 2], pa.int64()),
        "u8": pa.array([0, 255], pa.uint8()), "u16": pa.array([0, 65535], pa.uint16()), "u32": pa.array([0, 2**32 - 1], pa.uint32()),
        "u64": pa.array([0, 2**64 - 1], pa.uint64()),
        "ts_ms": pa.array([1, 2], TS("ms")), "ts_us": pa.array([1, 2], TS("us", tz="UTC")), "ts_ns": pa.array([1000, 2000], TS("ns")),
        "d1": pa.array([1, 2], pa.decimal128(1, 0)), "d9": pa.array([1, 2], pa.decimal128(9, 3)), "d18": pa.array([1, 2], pa.decimal128(18, 6)),
        "d38": pa.array([1, 2], pa.decimal128(38, 10)), "dt": pa.array([1, 2], pa.date32()), "s": pa.array(["a", "b"]), "b": pa.array([b"a", b"b"]),
        "f": pa.array([1.0, 2.0], pa.float32()),
    })
    path = str(tmp_path / "lt.parquet")
    pq.write_table(t, path, version=version, coerce_timestamps=coerce, store_decimal_as_integer=dec_int, allow_truncated_timestamps=True)
    d = _describe(path)
    leaves = [e for e in d["schema"] if e["num_children"] == 0]
    sch = pq.ParquetFile(path).schema
    for i, e in enumerate(leaves):
        col = sch.column(i)
        lt = col.logical_type.to_json()
        lt = json.loads(lt) if lt else {"Type": "None"}
        kind = lt["Type"].upper()
        assert e["name"] == col.name
        assert e["logical"] == _LK.get(kind, 6), (col.name, lt)
        if kind == "TIMESTAMP":
            assert e["ts_unit"] == _UNIT[lt["timeUnit"]] and e["ts_utc"] == lt["isAdjustedToUTC"], col.name
        if kind == "INT":
            assert (e["int_bits"], e["int_signed"]) == (lt["bitWidth"], lt["isSigned"]), col.name
        if kind == "DECIMAL":
            assert (e["precision"], e["scale"]) == (lt["precision"], lt["scale"]), col.name


@pytest.mark.parametrize("layout", parquet_pages.layouts(), ids=lambda x: x[0])
def test_hand_built_pages_read_back_through_pyarrow(tmp_path, layout):
    name, phys, required, pages, dictionary = layout
    path = str(tmp_path / f"{name}.parquet")
    want = parquet_pages.write(path, phys, required, pages, dictionary)
    got = pq.read_table(path)
    assert got["c"].to_pylist() == want
    assert got.schema.field("c").nullable == (not required)
    d = _describe(path)                                       # the engine's reader walks the same pages
    cm = d["row_groups"][0]["columns"][0]
    assert cm["page_values"] == len(want) and cm["data_pages"] == len(pages)
