"""What the reference engine hands on when it scans a Parquet column into a table type, in plain Python.

The reference reads the file with the third-party `parquet` crate, which gives the file's Arrow type, and then
AuronSchemaAdapter (datafusion-ext-plans/src/scan/mod.rs:103-160) turns every column into the table's type.  Arrow C++
(`pq.read_table`) stands in for the crate, as DESIGN section 4 states; the adapter's rules are restated below in Python
integers, one rule per branch, each next to where it comes from.

`read(path, schema)` gives, per table column, a list of canonical values (`canon`): ints for integers, dates, timestamps
(the count in the table's unit) and decimals (the unscaled integer), the IEEE bits of floats (every NaN as the string
"nan"), bytes for strings and binaries, None for NULL.  The engine's output goes through `canon_array` and must be equal.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

I64_MIN, I64_MAX = -2**63, 2**63 - 1
_UNIT_EXP = {"s": 0, "ms": 3, "us": 6, "ns": 9}
_INT_BITS = {pa.int8(): 8, pa.int16(): 16, pa.int32(): 32, pa.int64(): 64}
_UINT_BITS = {pa.uint8(): 8, pa.uint16(): 16, pa.uint32(): 32, pa.uint64(): 64}


def _float_bits(x: float, width: int):
    if x != x:
        return "nan"
    return int(np.array([x], dtype=np.float32 if width == 4 else np.float64).view(np.uint32 if width == 4 else np.uint64)[0])


def _fits_int(v: int, bits: int) -> bool:
    return -2**(bits - 1) <= v < 2**(bits - 1)


def convert_value(v, src: pa.DataType, dst: pa.DataType):
    """One value of the file's Arrow type `src` (as pq.read_table gives it, in Python form) -> canonical value of `dst`."""
    if v is None:
        return None
    # timestamps: the stored count (pq.read_table's python values are datetimes; callers pass the raw count)
    if pa.types.is_timestamp(src) and pa.types.is_timestamp(dst):
        # arrow cast.rs (Timestamp -> Timestamp): a finer unit multiplies with checked_mul, which the `safe` cast turns into NULL
        # on overflow; a coarser unit divides with Rust's `/`, which truncates toward zero (not Spark's floorDiv)
        d = _UNIT_EXP[dst.unit] - _UNIT_EXP[src.unit]
        if d >= 0:
            r = v * 10**d
            return r if I64_MIN <= r <= I64_MAX else None
        q = abs(v) // 10**-d
        return q if v >= 0 else -q
    if pa.types.is_timestamp(src) and dst == pa.int64():
        return v                                                  # arrow: Timestamp -> Int64 is the stored count
    if src == pa.int64() and pa.types.is_timestamp(dst):
        return v                                                  # arrow: Int64 -> Timestamp reinterprets the count in the target unit
    if (src in _INT_BITS or src in _UINT_BITS) and pa.types.is_decimal(dst):
        return v                                                  # scan/mod.rs:131-136: integer -> decimal is a value copy, no rescale
    if (src in _INT_BITS or src in _UINT_BITS) and dst in _INT_BITS:
        return v if _fits_int(v, _INT_BITS[dst]) else None        # arrow `safe` cast: NULL where the value does not fit
    if (src in _INT_BITS or src in _UINT_BITS) and dst == pa.float64():
        return _float_bits(float(v), 8)                           # |v| < 2^53: exact
    if pa.types.is_floating(src) and pa.types.is_floating(dst):
        return _float_bits(float(v), dst.bit_width // 8)          # float32 -> float64 is exact; same width is a copy
    if pa.types.is_decimal(src) and pa.types.is_decimal(dst):
        # arrow cast.rs (Decimal128 -> Decimal128, reached through cast_scan_input_array): a larger scale multiplies by 10^(s2-s1);
        # a value with more than p2 digits is NULL under `safe`
        assert dst.scale >= src.scale, "a narrower scale rounds; the engine rejects it"
        r = v * 10**(dst.scale - src.scale)
        return r if abs(r) < 10**dst.precision else None
    if pa.types.is_date32(src) and (pa.types.is_date32(dst) or dst == pa.int32()):
        return v
    if pa.types.is_date32(src) and dst == pa.int64():
        return v
    if (pa.types.is_string(src) or pa.types.is_binary(src) or pa.types.is_large_string(src)) and (pa.types.is_string(dst) or pa.types.is_binary(dst)):
        return v
    if pa.types.is_boolean(src) and pa.types.is_boolean(dst):
        return v
    raise TypeError(f"no reference rule for {src} -> {dst}")


def _raw_values(arr: pa.Array) -> list:
    """Python values with timestamps as their stored count and decimals as their unscaled integer."""
    t = arr.type
    if pa.types.is_timestamp(t) or pa.types.is_date32(t):
        return arr.cast(pa.int64() if pa.types.is_timestamp(t) else pa.int32()).to_pylist()
    if pa.types.is_decimal(t):
        return _decimal_unscaled(arr)
    if pa.types.is_string(t) or pa.types.is_large_string(t):
        return [None if v is None else v.encode() for v in arr.to_pylist()]
    return arr.to_pylist()


def _decimal_unscaled(arr: pa.Array) -> list:
    arr = arr.cast(pa.decimal128(arr.type.precision, arr.type.scale)) if not isinstance(arr.type, pa.Decimal128Type) else arr
    buf = arr.buffers()[1]
    raw = np.frombuffer(buf, dtype=np.uint64, count=2 * (len(arr) + arr.offset))[2 * arr.offset:]
    valid = arr.is_valid().to_pylist()
    out = []
    for i in range(len(arr)):
        if not valid[i]:
            out.append(None)
            continue
        u = int(raw[2 * i]) | (int(raw[2 * i + 1]) << 64)
        out.append(u - (1 << 128) if u >> 127 else u)
    return out


def canon_array(arr) -> list:
    """The engine's output column -> canonical values (see the module docstring)."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    t = arr.type
    if pa.types.is_floating(t):
        return [None if v is None else _float_bits(v, t.bit_width // 8) for v in arr.to_pylist()]
    return _raw_values(arr)


def read(path: str, schema: pa.Schema) -> dict[str, list]:
    """Canonical values of every column of `schema` as the reference scans `path` into it (missing columns are NULL, names
    match case-insensitively: scan/mod.rs:56-100)."""
    tab = pq.read_table(path)
    by_lower = {n.lower(): n for n in tab.column_names}
    out = {}
    for f in schema:
        name = f.name if f.name in tab.column_names else by_lower.get(f.name.lower())
        if name is None:
            out[f.name] = [None] * tab.num_rows
            continue
        col = tab[name].combine_chunks()
        src = col.type
        if src == f.type and not pa.types.is_floating(src):
            out[f.name] = _raw_values(col)                        # the same type: a copy
            continue
        vals = col.to_pylist() if pa.types.is_floating(src) else _raw_values(col)
        out[f.name] = [convert_value(v, src, f.type) for v in vals]
    return out
