"""The unfused Parquet decode has one path: every flat column of a batch is scouted by one shared pq_scout launch and decoded by one
pq_decode_pages launch of its own; a list column scouts and decodes its element values on its own.  The launch counts of a file with
every kind of column pin that, batch by batch.  And the host counts the non-null values of a nullable v1 PLAIN string page from its
definition levels with the bounds-checked level decoder: a level stream that ends before the page's values do fails the scan on the
host, before any kernel reads the page."""
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from auron_b200 import proto as P
from auron_b200 import runtime

pytestmark = pytest.mark.gpu

I32, I64, U = pa.int32(), pa.int64(), pa.string()


def _scan(path, schema):
    with runtime.Task(P.task_definition(P.parquet_scan(schema, [(path, os.path.getsize(path))], list(range(len(schema)))))) as task:
        out = pa.Table.from_batches(list(task), schema=task.schema)
        met = {}
        for _, op, name, v in task.metrics():
            met[(op, name)] = met.get((op, name), 0) + v
    return out, met


def _every_kind(n, seed):
    """a required int32, a nullable int64, a nullable dictionary string, a nullable PLAIN string and a list<int64>"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 5, n)
    xs = [None if i % 13 == 0 else [None if (i + k) % 6 == 0 else int(rng.integers(-10**12, 10**12)) for k in range(lens[i])] for i in range(n)]
    return pa.table({
        "i": pa.array(rng.integers(-2**31, 2**31, n).astype(np.int32)),
        "l": pa.array(rng.integers(-2**62, 2**62, n), I64, mask=rng.random(n) < 0.1),
        "ds": pa.array([f"d{x}" for x in rng.integers(0, 40, n)], U, mask=rng.random(n) < 0.1),
        "ps": pa.array([f"p{x}-{'y' * int(x % 17)}" for x in rng.integers(0, 10**9, n)], U, mask=rng.random(n) < 0.1),
        "xs": pa.array(xs, pa.list_(I64)),
    }).cast(pa.schema([pa.field("i", I32, nullable=False), pa.field("l", I64), pa.field("ds", U), pa.field("ps", U), pa.field("xs", pa.list_(I64))]))


@pytest.mark.parametrize("codec,page_version", [("SNAPPY", "1.0"), ("SNAPPY", "2.0"), ("ZSTD", "1.0")])
def test_one_scout_for_the_flat_columns_of_a_batch(tmp_path, monkeypatch, codec, page_version):
    rg = 3000
    t = _every_kind(10_000, 7)
    path = str(tmp_path / "kinds.parquet")
    pq.write_table(t, path, compression=codec, data_page_version=page_version, row_group_size=rg, data_page_size=4096, use_dictionary=["ds"])
    meta = pq.ParquetFile(path).metadata
    batches = meta.num_row_groups
    assert batches == 4
    for g in range(batches):   # the layout the counts below assume: dictionary pages for ds only
        encs = {meta.row_group(g).column(c).path_in_schema: meta.row_group(g).column(c).encodings for c in range(meta.num_columns)}
        assert any("DICTIONARY" in e for e in encs["ds"]), encs
        assert not any("DICTIONARY" in e for e in encs["ps"]), encs
    monkeypatch.setenv("AURON_GPU_CHUNK_ROWS", str(rg))   # one row group per batch
    monkeypatch.setenv("AURON_PROFILE", "1")
    got, met = _scan(path, t.schema)
    want = pq.read_table(path)
    assert got.num_rows == want.num_rows
    for c in want.column_names:
        assert got[c].to_pylist() == want[c].to_pylist(), c
    assert met[("__kernels__", "pq_scout.launches")] == 2 * batches, met   # the flat columns together, the list column alone
    assert met[("__kernels__", "pq_decode_pages.launches")] == 5 * batches, met


def test_level_stream_that_ends_early_fails_on_the_host(tmp_path):
    n = 200
    vals = [None if i < 16 and i % 2 else f"s{i:03d}" for i in range(n)]
    path = str(tmp_path / "levels.parquet")
    pq.write_table(pa.table({"s": pa.array(vals, U)}), path, compression="NONE", use_dictionary=False, data_page_version="1.0")
    col = pq.ParquetFile(path).metadata.row_group(0).column(0)
    data = bytearray(open(path, "rb").read())
    start, size = col.data_page_offset, col.total_compressed_size
    # the one data page ends the chunk: [header][u32 level length][levels][PLAIN values]; find where its body starts
    values_len = sum(4 + len(v) for v in vals if v is not None)
    body = [k for k in range(start + 1, start + 64) if k + 4 + struct.unpack_from("<I", data, k)[0] + values_len == start + size]
    assert len(body) == 1, body
    lv = body[0] + 4
    level_len = struct.unpack_from("<I", data, body[0])[0]
    # pyarrow writes the 16 alternating levels as one bit-packed run of 2 groups behind a one-byte header, then an RLE run of 184
    assert data[lv] == (2 << 1) | 1, data[lv:lv + level_len].hex()
    # the first run now claims 63 groups: more than the level section holds, while the section itself still lies inside the page
    data[lv] = (63 << 1) | 1
    assert 63 > level_len - 1
    bad = str(tmp_path / "short_levels.parquet")
    open(bad, "wb").write(bytes(data))
    with pytest.raises(runtime.AuronError, match="level stream ends early"):
        _scan(bad, pa.schema([pa.field("s", U)]))
