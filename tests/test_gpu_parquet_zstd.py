"""ZSTD and LZ4_RAW Parquet pages decompressed on the device (k_zstd.cu): the whole CPU corpus of test_zstd_host.py as page bodies
of hand-built files, pyarrow-written files of every type and layout against the reference reader, where each page is
decompressed (the pages_decompressed_device / _host metrics), list columns, the fused scan -> filter -> aggregate pass, several
files, row groups and batches, file images in host memory and in HBM, and damaged pages."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import test_gpu_parquet_edges as E
import test_zstd_host as H
import zstd_frames as Z
import zstd_pages
from auron_b200 import proto as P
from auron_b200 import runtime

pytestmark = pytest.mark.gpu

I64 = pa.int64()


def _task(plan, env=None):
    env = env or {}
    old = {k: os.environ.get(k) for k in env}
    try:
        for k, v in env.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        with runtime.Task(P.task_definition(plan)) as task:
            out = pa.Table.from_batches(list(task), schema=task.schema)
            met = {}
            for _, op, name, v in task.metrics():
                met[(op, name)] = met.get((op, name), 0) + v
        return out, met
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _scan(paths, schema, env=None, sizes=None):
    files = [(p, sizes[i] if sizes else os.path.getsize(p)) for i, p in enumerate(paths)]
    return _task(P.parquet_scan(schema, files, list(range(len(schema)))), env)


def _where(met):
    return met.get(("ParquetExec", "pages_decompressed_device"), 0), met.get(("ParquetExec", "pages_decompressed_host"), 0)


def test_cpu_corpus_as_page_bodies(tmp_path):
    bodies = []
    for name, frame, data in H.corpus():
        if len(data) % 8 == 0 and data:   # (an empty page at the end of a chunk is never visited)
            bodies.append((name, frame, data))
    assert len(bodies) > 40
    schema = pa.schema([pa.field("c", I64, nullable=False)])
    # one file per frame would be slow: a few frames per file, each its own page
    for g in range(0, len(bodies), 12):
        grp = bodies[g:g + 12]
        path = str(tmp_path / f"corpus{g}.parquet")
        zstd_pages.write(path, [(f, len(d)) for _, f, d in grp])
        got, met = _scan([path], schema)
        want = np.concatenate([np.frombuffer(d, np.int64) for _, _, d in grp]) if grp else np.zeros(0, np.int64)
        assert got.num_rows == len(want), [n for n, _, _ in grp]
        assert np.array_equal(got["c"].to_numpy(), want), [n for n, _, _ in grp]
        assert _where(met) == (len(grp), 0), met


def _lz4_block(data):
    """a raw LZ4 block of literals and matches, written here (liblz4 through pyarrow's codec)"""
    return pa.compress(data, codec="lz4_raw", asbytes=True)


def test_lz4_raw_page_bodies(tmp_path):
    sh = Z.shapes(400_000, 5)
    pages = [(sh[k][:n - n % 8], k) for k, n in (("int64", 80_000), ("runs", 131_072), ("period", 400_000), ("noisy", 8), ("text", 65_536))]
    path = str(tmp_path / "lz4.parquet")
    zstd_pages.write(path, [(_lz4_block(d), len(d)) for d, _ in pages], codec=zstd_pages.CODEC_LZ4_RAW)
    got, met = _scan([path], pa.schema([pa.field("c", I64, nullable=False)]))
    want = np.concatenate([np.frombuffer(d, np.int64) for d, _ in pages])
    assert np.array_equal(got["c"].to_numpy(), want)
    assert _where(met) == (len(pages), 0)


@pytest.mark.parametrize("codec", ["ZSTD", "LZ4_RAW"])
def test_damaged_page_names_the_codec(tmp_path, codec):
    d = Z.shapes(64_000, 6)["int64"]
    if codec == "ZSTD":
        good = Z.compress(d, level=3)
        bad = bytearray(good)
        bad[len(bad) // 2] ^= 0xFF   # inside the sequences: an impossible stream
        body = [(bytes(good), len(d)), (bytes(bad[:-3]), len(d))]
        c = zstd_pages.CODEC_ZSTD
    else:
        good = _lz4_block(d)
        bad = bytearray(good)
        bad[-1] ^= 0xFF
        bad = bad[:-2]
        body = [(bytes(good), len(d)), (bytes(bad), len(d))]
        c = zstd_pages.CODEC_LZ4_RAW
    path = str(tmp_path / "bad.parquet")
    zstd_pages.write(path, body, codec=c)
    with pytest.raises(runtime.AuronError, match="corrupt " + codec + " page"):
        _scan([path], pa.schema([pa.field("c", I64, nullable=False)]))


@pytest.mark.parametrize("codec,level", [("ZSTD", 1), ("ZSTD", 3), ("ZSTD", 9), ("ZSTD", 19), ("LZ4_RAW", None)])
@pytest.mark.parametrize("layout", [("1.0", True, False), ("2.0", True, False), ("1.0", False, False), ("2.0", False, True)],
                         ids=["v1-dict-nullable", "v2-dict-nullable", "v1-plain-nullable", "v2-plain-required"])
def test_types_at_their_edges(tmp_path, codec, level, layout):
    page_version, dict_, required = layout
    t = E._edge_table(1500, "none" if required else "alternating")
    if required:
        t = t.cast(pa.schema([pa.field(f.name, f.type, nullable=False) for f in t.schema]))
    path = str(tmp_path / "edges.parquet")
    kw = {"compression_level": level} if codec == "ZSTD" else {}
    pq.write_table(t, path, use_dictionary=dict_, version="2.6", data_page_version=page_version, compression=codec, row_group_size=700,
                   data_page_size=2048, write_batch_size=64, store_decimal_as_integer=True, **kw)
    for schema in E._read_schemas(t.schema):
        E._check(path, schema)
    # where each page went: the host decompresses exactly the nullable v1 PLAIN string / binary pages
    got, met = _scan([path], E._read_schemas(t.schema)[0])
    nullable_v1_plain = not required and page_version == "1.0" and not dict_
    _assert_where(met, path, page_version, lambda ch: ch["type"] == 6 and nullable_v1_plain)


def _assert_where(met, path, page_version, on_host):
    """the host decompresses exactly the pages of the chunks on_host() names; the device all other compressed pages (a v2 page may be
    stored uncompressed: then neither)"""
    total, host = _count_pages(path, on_host)
    dev, got_host = _where(met)
    assert got_host == host, (met, total, host)
    if page_version == "1.0":
        assert dev == total - host, (met, total, host)
    else:
        assert 0 < dev <= total - host, (met, total, host)


@pytest.mark.parametrize("page_mb", [1, 8])
def test_large_pages(tmp_path, page_mb):
    rng = np.random.default_rng(page_mb)
    n = 2_500_000
    t = pa.table({"k": pa.array(np.cumsum(rng.integers(0, 50, n)), I64), "v": pa.array(rng.integers(0, 1 << 20, n).astype(np.int32))})
    path = str(tmp_path / "big.parquet")
    pq.write_table(t, path, compression="ZSTD", use_dictionary=False, data_page_size=page_mb << 20, row_group_size=n)
    got, met = _scan([path], t.schema)
    assert got["k"].to_numpy().tolist() == t["k"].to_numpy().tolist()
    assert np.array_equal(got["v"].to_numpy(), t["v"].to_numpy())
    assert _where(met) == (_count_pages(path, lambda ch: False)[0], 0)


@pytest.mark.parametrize("codec", ["ZSTD", "LZ4_RAW"])
@pytest.mark.parametrize("page_version", ["1.0", "2.0"])
def test_list_columns(tmp_path, codec, page_version):
    # v2 list pages carry their levels outside the body: device; v1 list pages are decompressed on the host, which counts their levels
    rng = np.random.default_rng(11)
    n = 4000
    lens = rng.integers(0, 6, n)
    vals = [None if i % 17 == 0 else [None if (i + k) % 7 == 0 else int(rng.integers(-1000, 1000)) for k in range(lens[i])] for i in range(n)]
    t = pa.table({"id": pa.array(np.arange(n), I64), "xs": pa.array(vals, pa.list_(I64)),
                  "ss": pa.array([None if v is None else [str(x) for x in v if x is not None] for v in vals], pa.list_(pa.string()))})
    path = str(tmp_path / "lists.parquet")
    pq.write_table(t, path, compression=codec, data_page_version=page_version, data_page_size=1024, row_group_size=1500, use_dictionary=False)
    got, met = _scan([path], t.schema)
    exp = pq.read_table(path)
    for c in t.column_names:
        assert got[c].to_pylist() == exp[c].to_pylist(), c
    _assert_where(met, path, page_version, lambda ch: page_version == "1.0" and ch["path"] != "id")


def _config2(n, seed):
    rng = np.random.default_rng(seed)
    return pa.table({"ss_item_sk": pa.array(rng.integers(1, 20_000, n).astype(np.int32)),
                     "ss_quantity": pa.array(rng.integers(1, 101, n).astype(np.int32), mask=rng.random(n) < 0.03),
                     "ss_sold_date_sk": pa.array(rng.integers(2450816, 2452642, n).astype(np.int32), mask=rng.random(n) < 0.04)})


def _agg_plan(paths, schema):
    scan = P.parquet_scan(schema, [(p, os.path.getsize(p)) for p in paths], [0, 1, 2])
    flt = P.filter_(scan, [P.binary("GtEq", P.col("ss_sold_date_sk"), P.lit(2451000, pa.int32())),
                           P.binary("Lt", P.col("ss_sold_date_sk"), P.lit(2452000, pa.int32()))])
    return P.agg(flt, [P.try_cast(P.col("ss_item_sk"), I64)], ["item"],
                 [P.agg_expr("SUM", [P.col("ss_quantity")], I64), P.agg_expr("COUNT", [P.col("ss_quantity")], I64)], ["s", "c"], ["PARTIAL", "PARTIAL"])


def _rows(t):
    return sorted(zip(*[c.to_pylist() for c in t.columns]), key=lambda r: tuple((0, 0) if v is None else (1, v) for v in r))


@pytest.mark.parametrize("codec,level", [("ZSTD", 1), ("ZSTD", 3), ("LZ4_RAW", None)])
def test_fused_scan_filter_aggregate(tmp_path, codec, level):
    t = _config2(600_000, 12)
    paths = []
    for i in range(2):
        paths.append(str(tmp_path / f"c2_{i}.parquet"))
        part = t.slice(i * 300_000, 300_000)
        pq.write_table(part, paths[-1], compression=codec, use_dictionary=True, row_group_size=100_000,
                       **({"compression_level": level} if level else {}))
    fused, met = _task(_agg_plan(paths, t.schema))
    plain, met0 = _task(_agg_plan(paths, t.schema), {"AURON_DISABLE_FUSED_SCAN_AGG": "1"})
    assert met.get(("ParquetExec", "fused_batches"), 0) > 0, met
    assert met0.get(("ParquetExec", "fused_batches"), 0) == 0
    assert _rows(fused) == _rows(plain)
    assert _where(met)[1] == 0 and _where(met)[0] > 0, met
    # and against pyarrow
    ref = pa.concat_tables([pq.read_table(p) for p in paths])
    d = ref["ss_sold_date_sk"].to_numpy(zero_copy_only=False)
    keep = ~np.isnan(d.astype(float)) & (np.nan_to_num(d.astype(float)) >= 2451000) & (np.nan_to_num(d.astype(float)) < 2452000)
    sub = ref.filter(pa.array(keep))
    g = sub.group_by("ss_item_sk").aggregate([("ss_quantity", "sum"), ("ss_quantity", "count")])
    want = sorted((int(k), s, c) for k, s, c in zip(g["ss_item_sk"].to_pylist(), g["ss_quantity_sum"].to_pylist(), g["ss_quantity_count"].to_pylist()))
    assert _rows(fused) == want


@pytest.mark.parametrize("image", ["file", "host", "device"])
@pytest.mark.parametrize("codec", ["ZSTD", "LZ4_RAW"])
def test_files_row_groups_batches_and_images(tmp_path, image, codec):
    rng = np.random.default_rng(13)
    tables, paths = [], []
    for i in range(3):
        n = 7000 + 1000 * i
        t = pa.table({"a": pa.array(rng.integers(-10**12, 10**12, n), I64, mask=rng.random(n) < 0.1),
                      "s": pa.array([f"v{x}" for x in rng.integers(0, 300, n)]),
                      "d": pa.array(rng.random(n))})
        p = str(tmp_path / f"m{i}.parquet")
        pq.write_table(t, p, compression=codec, row_group_size=2500, data_page_size=4096, data_page_version=("1.0", "2.0")[i % 2])
        tables.append(t)
        paths.append(p)
    names, sizes = paths, None
    if image != "file":
        names = [f"{image}://zstd/{i}" for i in range(3)]
        sizes = [os.path.getsize(p) for p in paths]
        keep = []
        for nm, p in zip(names, paths):
            data = open(p, "rb").read()
            if image == "device":
                runtime.put_device_file(nm, data)
            else:
                buf = np.frombuffer(data, np.uint8).copy()
                keep.append(buf)
                runtime.put_host_file(nm, buf)
    try:
        got, met = _scan(names, tables[0].schema, {"AURON_GPU_CHUNK_ROWS": "3000"}, sizes)
    finally:
        for nm in names if image != "file" else []:
            (runtime.drop_device_file if image == "device" else runtime.drop_host_file)(nm)
    want = pa.concat_tables([pq.read_table(p) for p in paths])
    for c in want.column_names:
        assert got[c].to_pylist() == want[c].to_pylist(), c
    assert _where(met)[0] > 0


def _count_pages(path, on_host):
    """(all pages, pages of the chunks for which on_host(chunk) holds), from the engine's own walk of the page headers"""
    import ctypes as C
    import json
    L = runtime.lib()
    L.auron_b200_parquet_describe.restype = C.c_int64
    L.auron_b200_parquet_describe.argtypes = [C.c_char_p, C.c_char_p, C.c_int64]
    buf = C.create_string_buffer(1 << 24)
    assert L.auron_b200_parquet_describe(path.encode(), buf, len(buf)) > 0
    total = host = 0
    for rg in json.loads(buf.value.decode())["row_groups"]:
        for ch in rg["columns"]:
            total += ch["data_pages"] + ch["dictionary_pages"]
            host += ch["data_pages"] if on_host(ch) else 0
    return total, host
