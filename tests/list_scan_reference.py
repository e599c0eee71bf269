"""What the reference hands on when it scans a Parquet LIST column into a table list type, in plain Python.

arrow-rs reads the list with its offsets and NULL rows; AuronSchemaAdapter casts its elements to the table's element type
(datafusion-ext-plans/src/scan/mod.rs:143-156, schema_adapter_cast_column), one element at a time with the flat rules, which
scan_reference.convert_value restates.  `read(path, schema)` gives flat columns as scan_reference.read does and list columns as
None (a NULL list) or a list of canonical element values; `canon_column` turns the engine's output into the same form.
"""
from __future__ import annotations

import pyarrow as pa
import pyarrow.parquet as pq

import scan_reference as R


def _rows(col: pa.Array, elems: list) -> list:
    off = col.offsets.to_pylist()
    valid = col.is_valid().to_pylist()
    return [list(elems[off[i]:off[i + 1]]) if valid[i] else None for i in range(len(col))]


def _flat_values(col: pa.Array) -> pa.Array:
    off = col.offsets.to_pylist()
    return col.values.slice(off[0], off[-1] - off[0]) if len(col) else col.values.slice(0, 0)


def read(path: str, schema: pa.Schema) -> dict[str, list]:
    flat = pa.schema([f for f in schema if not pa.types.is_list(f.type)])
    out = R.read(path, flat)
    tab = pq.read_table(path)
    by_lower = {n.lower(): n for n in tab.column_names}
    for f in schema:
        if not pa.types.is_list(f.type):
            continue
        name = f.name if f.name in tab.column_names else by_lower.get(f.name.lower())
        if name is None:
            out[f.name] = [None] * tab.num_rows
            continue
        col = tab[name].combine_chunks()
        src, dst = col.type.value_type, f.type.value_type
        vals = _flat_values(col)
        raw = vals.to_pylist() if pa.types.is_floating(src) else R._raw_values(vals)
        if src == dst and not pa.types.is_floating(src):
            conv = raw
        else:
            conv = [R.convert_value(v, src, dst) for v in raw]
        off0 = col.offsets[0].as_py() if len(col) else 0
        out[f.name] = _rows(col, [None] * off0 + conv)
    return out


def canon_column(arr) -> list:
    """the engine's output column (flat or list) -> canonical values"""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    if not pa.types.is_list(arr.type):
        return R.canon_array(arr)
    vals = _flat_values(arr)
    off0 = arr.offsets[0].as_py() if len(arr) else 0
    return _rows(arr, [None] * off0 + R.canon_array(vals))
