"""The shuffle byte format end to end against the plain-Python references of shuffle_reference.py: ShuffleWriterExec and
IpcWriterExec output must be the bytes the reference's write_batch would write (batch_serde.rs), in LZ4 frames / blocks that obey
the format's end rules (a reader on the CPU engine is lz4_flex, which may not check them), and IpcReaderExec must read frames shaped
like lz4_flex's FrameEncoder output (independent 64 KB blocks, liblz4's parse) on the device path.  Values are compared by their
bits (key_reference canonical form), never with a float ==.

  (a) writer x every column type x partition sizes at the warp-chunk, validity-byte and varint edges x codec x chunking
  (b) the fast and row-wise serde kernels write the same bytes
  (c) the GPU LZ4 compressor at block edges, on crafted bytes
  (d) the reader on both decode paths, on the writer's files and on reference-shaped frames
  (e) IpcWriterExec's consumer blocks"""
import functools
import random
import struct

import numpy as np
import pyarrow as pa
import pytest

import key_reference as R
import oracle
import shuffle_reference as S
from auron_b200 import proto as P
from auron_b200 import runtime
from test_gpu_key_edges import BITMAPS, from_arrow, to_arrow, with_env

pytestmark = pytest.mark.gpu

# partition sizes across the 128-row warp chunks of serde_fixed_kernel, the byte edges of the validity sections and the varint
# row count's 1 -> 2 -> 3 byte steps
SIZES = [0, 0, 1, 2, 3, 4, 5, 7, 8, 9, 31, 32, 33, 127, 128, 129, 255, 256, 257, 16383, 16384, 16385]
CODECS = {"gpu_lz4": {"AURON_IO_COMPRESSION_CODEC": "lz4"},
          "host_lz4": {"AURON_IO_COMPRESSION_CODEC": "lz4", "AURON_HOST_LZ4": "1"},
          "zstd": {"AURON_IO_COMPRESSION_CODEC": "zstd"}}
# (name, reference type); the extra columns: a Null-typed column and two columns whose every value is NULL
EXTRA = [("nul", "null"), ("allnull_i16", "int16"), ("allnull_utf8", "utf8")]
SCHEMA = [(t, t) for t in R.TYPES] + EXTRA + [("row", "int64")]
TYPES = [ty for _, ty in SCHEMA]
GPU_HEADER = bytes([0x60, 0x40, 0x82])                  # FLG (v1, independent blocks), BD (64 KB), HC


# -------------------------------------------------------------------------------------------- inputs
@functools.lru_cache(maxsize=None)
def every_type_table(n: int, off: int = 0, seed: int = 1):
    """n rows of every type (edge values, the three bitmap shapes), the extra columns and `row` = 0..n-1; the arrays are
    sliced at `off`.  -> (table, {name: canonical values})"""
    arrs, vals = {}, {}
    for i, t in enumerate(R.TYPES):
        bitmap = BITMAPS[i % 3]
        v = R.edge_column(t, n + off, seed + i, null_rate=0.05 if bitmap == "nulls" else 0.0)
        vals[t], arrs[t] = v[off:], to_arrow(v, t, bitmap != "no_bitmap").slice(off)
    arrs["nul"], vals["nul"] = pa.nulls(n + off).slice(off), [None] * n
    for name, t in EXTRA[1:]:
        arrs[name], vals[name] = to_arrow([None] * (n + off), t).slice(off), [None] * n
    arrs["row"], vals["row"] = pa.array(np.arange(-off, n), type=pa.int64()).slice(off), list(range(n))
    return pa.table(arrs), vals


def range_bounds(sizes):
    """bounds of a range partitioning on `row` that gives partitions of exactly these sizes (a key equal to a bound stays below it)"""
    cum = np.cumsum(sizes)
    return [int(c) - 1 for c in cum[:-1]]


def write_shuffle(tmp_path, table, repartition, env, chunk=None, tag="s"):
    data, index = str(tmp_path / f"{tag}.data"), str(tmp_path / f"{tag}.index")
    plan = P.shuffle_writer(P.ffi_reader(table.schema, "t"), repartition, data, index)
    env = dict(env, **({"AURON_GPU_CHUNK_ROWS": str(chunk)} if chunk else {}))

    def go():
        with runtime.Task(P.task_definition(plan), {"t": table.to_batches(max_chunksize=chunk or table.num_rows)}) as task:
            assert list(task) == []
    with_env(env, go)
    idx = open(index, "rb").read()
    return data, open(data, "rb").read(), list(struct.unpack(f"<{len(idx) // 8}q", idx))


def write_every_type(tmp_path, codec, chunking):
    n = sum(SIZES)
    off = 3 if chunking == "sliced" else 0
    table, vals = every_type_table(n, off)
    chunk = {"one_chunk": None, "chunks": 5000, "sliced": 7001}[chunking]
    rep = P.range_repartition([P.sort_expr(P.col("row"), True, True)], len(SIZES), [(range_bounds(SIZES), pa.int64())])
    path, data, offsets = write_shuffle(tmp_path, table, rep, CODECS[codec], chunk, tag=f"{codec}_{chunking}")
    starts = np.concatenate([[0], np.cumsum(SIZES)])
    return table, vals, path, data, offsets, [list(range(starts[p], starts[p + 1])) for p in range(len(SIZES))]


# -------------------------------------------------------------------------------------------- decoding with the references
def gpu_frame_payload(info, stats):
    """the content of one frame written by the GPU compressor: the fixed header, independent 64 KB blocks, every compressed block
    decoded by the strict decoder and by liblz4 to the same bytes, and smaller than what it holds"""
    assert bytes([info["flg"], info["bd"], info["hc"]]) == GPU_HEADER
    out = b""
    for i, (stored, blk) in enumerate(info["blocks"]):
        last = i == len(info["blocks"]) - 1
        if stored:
            raw = blk
        else:
            raw, _ = S.lz4_block_decode(blk, expected_len=None if last else 65536, stats=stats)
            assert len(blk) < len(raw), "a compressed block that is not smaller than its content must be stored"
            assert bytes(pa.decompress(blk, decompressed_size=len(raw), codec="lz4_raw")) == raw
        assert len(raw) == 65536 or (last and 0 < len(raw) <= 65536)
        out += raw
    return out


def segment_payload(seg: bytes, codec: str, stats=None) -> bytes:
    stats = stats if stats is not None else S.new_stats()
    out = b""
    for st in S.split_streams(seg):
        if codec == "zstd":
            assert struct.unpack_from("<I", st, 4)[0] == 0xFD2FB528
            out += pa.CompressedInputStream(pa.BufferReader(st[4:]), "zstd").read()
            continue
        info = S.lz4_frame_blocks(st)
        if codec == "gpu_lz4":
            out += gpu_frame_payload(info, stats)
        else:
            got = S.lz4_frame_decode(info, stats)
            assert got == pa.CompressedInputStream(pa.BufferReader(st[4:]), "lz4").read()
            out += got
    return out


def check_payload(payload: bytes, vals: dict, schema=SCHEMA):
    """every batch of a partition's payload is byte for byte write_batch of the rows it holds (in the order its `row` column gives,
    with the has_nulls flags it chose; a NULL under has_nulls = 0 fails write_batch) -> (rows, batches)"""
    types = [ty for _, ty in schema]
    batches = S.read_sections(payload, types)
    rows = []
    for b in batches:
        rws = b["cols"][len(schema) - 1]
        exp = [(ty, [vals[name][r] for r in rws]) for name, ty in schema]
        assert payload[b["start"]:b["end"]] == S.write_batch(exp, b["has_nulls"]), f"batch of {b['n']} rows"
        rows += rws
    return rows, batches


def check_files(data, offsets, codec, vals, expected_rows, stats):
    nparts = len(expected_rows)
    assert len(offsets) == nparts + 1 and offsets[0] == 0 and offsets[-1] == len(data)
    assert all(a <= b for a, b in zip(offsets, offsets[1:]))
    payloads = []
    for p in range(nparts):
        seg = data[offsets[p]:offsets[p + 1]]
        if not expected_rows[p]:
            assert seg == b"", p                             # empty partitions write nothing
            payloads.append(b"")
            continue
        payload = segment_payload(seg, codec, stats)
        rows, batches = check_payload(payload, vals)
        assert sorted(rows) == sorted(expected_rows[p]) and len(set(rows)) == len(rows), p
        payloads.append(payload)
    return payloads


# -------------------------------------------------------------------------------------------- (a) writer x every type
@pytest.mark.parametrize("codec,chunking", [("gpu_lz4", "one_chunk"), ("gpu_lz4", "chunks"), ("gpu_lz4", "sliced"), ("host_lz4", "one_chunk"),
                                            ("host_lz4", "chunks"), ("zstd", "one_chunk"), ("zstd", "chunks")])
def test_writer_every_type_at_partition_size_edges(tmp_path, codec, chunking):
    table, vals, _, data, offsets, expected = write_every_type(tmp_path, codec, chunking)
    stats = S.new_stats()
    payloads = check_files(data, offsets, codec, vals, expected, stats)
    if chunking != "one_chunk":
        big = [p for p, s in enumerate(SIZES) if s > 10_000]
        assert all(len(S.read_sections(payloads[p], TYPES)) >= 3 for p in big)   # several device chunks per large partition
        return
    # one device chunk: the partitions' payloads are concatenated in order in one serialisation buffer, so every byte plane's
    # offset in that buffer is known; the fast kernel's full 128-row chunks must start at every alignment for every width
    align = {2: set(), 4: set(), 8: set(), 16: set()}
    base = 0
    for payload in payloads:
        for b in S.read_sections(payload, TYPES):
            for ty, vo in zip(TYPES, b["values_off"]):
                w = S.FIXED_WIDTH.get(ty)
                if w in align and b["n"] >= 128:
                    align[w] |= {(base + vo + k * b["n"]) & 3 for k in range(w)}
        base += len(payload)
    assert all(a == {0, 1, 2, 3} for a in align.values()), align
    if codec == "gpu_lz4":
        assert stats["matches"] > 0 and stats["blocks"] > 0


def test_writer_hash_partitioned_every_type(tmp_path):
    # hash partitioning on a mixed key: rows reach the serde kernels in partition order, not in `row` order
    n, nparts = 30_000, 7
    table, vals = every_type_table(n, 0, seed=7)
    _, data, offsets = write_shuffle(tmp_path, table, P.hash_repartition([P.col("int32"), P.col("utf8")], nparts), CODECS["gpu_lz4"], 12_000)
    pid = oracle.partition_ids([table["int32"].combine_chunks(), table["utf8"].combine_chunks()], nparts)
    check_files(data, offsets, "gpu_lz4", vals, [np.nonzero(pid == p)[0].tolist() for p in range(nparts)], None)


# -------------------------------------------------------------------------------------------- (b) fast vs row-wise serde
@pytest.mark.parametrize("chunking", ["one_chunk", "sliced"])
def test_fast_and_rowwise_serde_write_the_same_bytes(tmp_path, chunking):
    # AURON_SERDE_ROWWISE=1 sends widths 2 / 4 / 8 / 16 through serde_column_kernel instead of serde_fixed_kernel
    outs = []
    for rowwise in (False, True):
        env = dict(CODECS["zstd"], **({"AURON_SERDE_ROWWISE": "1"} if rowwise else {}))
        n = sum(SIZES)
        off = 3 if chunking == "sliced" else 0
        table, vals = every_type_table(n, off)
        rep = P.range_repartition([P.sort_expr(P.col("row"), True, True)], len(SIZES), [(range_bounds(SIZES), pa.int64())])
        _, data, offsets = write_shuffle(tmp_path, table, rep, env, 7001 if off else None, tag=f"rw{rowwise}")
        outs.append([segment_payload(data[a:b], "zstd") for a, b in zip(offsets, offsets[1:])])
    assert outs[0] == outs[1]
    for payload in outs[1]:
        if payload:
            check_payload(payload, vals)


# -------------------------------------------------------------------------------------------- (c) GPU LZ4 compressor at block edges
def _rng_bytes(rng, k):
    return bytes(rng.randrange(256) for _ in range(k))


def _lz_hash(b4: bytes) -> int:
    return ((int.from_bytes(b4, "little") * 2654435761) & 0xFFFFFFFF) >> 20


def _unique_hash(data: bytes, pos: int, upto: int) -> bool:
    """the compressor's 4096-entry position table keeps `pos` until `upto` (no other scanned position with the same hash)"""
    h = _lz_hash(data[pos:pos + 4])
    return all(_lz_hash(data[q:q + 4]) != h for q in range(upto) if q != pos)


def _header(clen: int) -> bytes:
    return b"\x01\x00" + struct.pack("<I", clen)         # 1 row, has_nulls 0, the one string length (four 1-byte planes)


def crafted_contents():
    """name -> (binary value, what the compressed stream must show).  The compressor's input is _header(len) + value."""
    rng = random.Random(11)
    out = {}
    for size in list(range(6, 14)) + [65535, 65536, 65537, 2 * 65536 + 1]:
        c = size - 6
        out[f"zeros_{size}"] = (bytes(c), None)
        for per in (2, 3, 5, 7):
            out[f"period{per}_{size}"] = ((_rng_bytes(rng, per) * (c // per + 1))[:c], None)
        out[f"random_{size}"] = (_rng_bytes(rng, c), "stored")
        pat = _rng_bytes(rng, 64)                       # equal up to the last byte: the match is cut at the last-literals limit
        out[f"tail_equal_{size}"] = ((_rng_bytes(rng, 40) + pat * (c // 64 + 1))[:c], None)
    while True:                                          # a literal run of exactly 15 + 255 bytes, then a repeat of its start
        x = _rng_bytes(rng, 264)
        data = _header(264 + 100 + 20) + x + x[:100] + _rng_bytes(rng, 20)
        if _unique_hash(data, 6, 256):
            out["literal_270"] = (data[6:], ("literal", 270))
            break
    for k in (0, 1, 2):                                  # a match of 4 + 15 + 255 k bytes: the extension ends in 255 x k, 0
        mlen = 19 + 255 * k
        while True:
            a = _rng_bytes(rng, 300)
            rep = (a * 3)[:mlen]
            brk = bytes([(a * 3)[mlen] ^ 0xFF])
            value = a + rep + brk + _rng_bytes(rng, 40)
            data = _header(len(value)) + value
            if _unique_hash(data, 6, 288):
                out[f"match_ext_{k}"] = (value, ("match", mlen))
                break
    while True:                                          # the farthest match a 64 KB block allows: 65523 back, to the header
        r = _rng_bytes(rng, 34)
        data = bytearray(_header(65530) + r + bytes(65523 - 40))
        data += data[:8] + _rng_bytes(rng, 5)
        if _unique_hash(bytes(data), 0, 64) and _lz_hash(data[:4]) != 0:
            assert len(data) == 65536
            out["offset_65523"] = (bytes(data[6:]), ("offset", 65523))
            break
    return out


def tiny_tables():
    """compressor inputs of 1 to 5 bytes (below the 6 bytes of a one-row binary batch)"""
    return {1: pa.table({"z": pa.nulls(1)}), 2: pa.table({"z": pa.nulls(128)}), 3: pa.table({"i": pa.array([-1], pa.int8())}),
            4: pa.table({"i": pa.array([0x1234], pa.int16())}), 5: pa.table({"i": pa.array([None], pa.int16())})}


def _tiny_schema(table):
    return [(f.name, {"null": "null", "int8": "int8", "int16": "int16"}[str(f.type)]) for f in table.schema]


def write_single(tmp_path, table, tag):
    return write_shuffle(tmp_path, table, P.single_repartition(1), CODECS["gpu_lz4"], tag=tag)


def check_single_frame(data, offsets, expected_payload, stats):
    assert offsets == [0, len(data)]
    streams = S.split_streams(data)
    assert len(streams) == 1
    info = S.lz4_frame_blocks(streams[0])
    assert gpu_frame_payload(info, stats) == expected_payload
    for stored, blk in info["blocks"]:
        raw_len = len(blk) if stored else len(S.lz4_block_decode(blk)[0])
        if raw_len <= 13:
            assert stored                                # no match fits: the sequence is longer than its content
    return info


CRAFTED = crafted_contents()


@pytest.mark.parametrize("name", sorted(CRAFTED))
def test_gpu_lz4_compressor_on_crafted_blocks(tmp_path, name):
    value, want = CRAFTED[name]
    table = pa.table({"b": to_arrow([value], "binary", bitmap=False)})
    _, data, offsets = write_single(tmp_path, table, "c")
    stats = S.new_stats()
    exp = S.write_batch([("binary", [value])], [0])
    assert exp[:6] == _header(len(value))
    info = check_single_frame(data, offsets, exp, stats)
    blocks = info["blocks"]
    assert len(blocks) == (len(exp) + 65535) // 65536
    if want == "stored":
        assert all(s for s, _ in blocks)
    elif want is not None:
        kind, v = want
        assert v in {"literal": stats["literal_lengths"], "match": stats["match_lengths"]}.get(kind, {stats["max_offset"]}), (want, stats)
    if name.startswith(("zeros", "period")) and len(exp) >= 65536:
        assert not blocks[0][0]
        if name.startswith("zeros"):
            assert len(blocks[0][1]) < 1024              # an all-zero 64 KB block


def test_gpu_lz4_compressor_on_tiny_inputs(tmp_path):
    for size, table in tiny_tables().items():
        schema = _tiny_schema(table)
        vals = [(ty, [None] * table.num_rows if ty == "null" else table[name].to_pylist()) for name, ty in schema]
        exp = S.write_batch(vals, [None if ty == "null" else int(table[name].null_count > 0) for name, ty in schema])
        assert len(exp) == size
        _, data, offsets = write_single(tmp_path, table, f"t{size}")
        info = check_single_frame(data, offsets, exp, S.new_stats())
        assert info["blocks"] == [(True, exp)]


# -------------------------------------------------------------------------------------------- (d) the reader on both decode paths
DECODE = {"device_path": {}, "host_path": {"AURON_HOST_LZ4_DECODE": "1"}}


def read_back(schema: pa.Schema, blocks, decode):
    def go():
        with runtime.Task(P.task_definition(P.ipc_reader(schema, "in")), shuffle_blocks={"in": blocks}) as task:
            got = pa.Table.from_batches(list(task), schema=task.schema)
            names = {name for _, op, name, _ in task.metrics() if op == "IpcReaderExec"}
        return got, names
    return with_env(DECODE[decode], go)


def check_read(got, vals, schema=SCHEMA, rows=None):
    rws = got["row"].to_pylist() if rows is None else rows
    for name, ty in schema:
        if ty == "null":
            assert got[name].null_count == got.num_rows
            continue
        assert from_arrow(got[name], ty) == [vals[name][r] for r in rws], name
    return rws


@pytest.mark.parametrize("decode", ["device_path", "host_path"])
@pytest.mark.parametrize("codec,chunking", [("gpu_lz4", "one_chunk"), ("gpu_lz4", "chunks"), ("gpu_lz4", "sliced"), ("host_lz4", "chunks"), ("zstd", "chunks")])
def test_reader_reads_every_type_writer_files(tmp_path, codec, chunking, decode):
    table, vals, path, data, offsets, expected = write_every_type(tmp_path, codec, chunking)
    for p in range(len(SIZES)):
        if not expected[p]:
            continue
        got, names = read_back(table.schema, [(path, offsets[p], offsets[p + 1] - offsets[p])], decode)
        assert sorted(check_read(got, vals)) == expected[p]
        # decompress_ns is recorded only by the host decode path (shuffle_reader.cc); the device path takes LZ4 frames with
        # independent blocks, which liblz4 also writes when a partition's payload fits in one block
        seg = data[offsets[p]:offsets[p + 1]]
        independent = codec != "zstd" and all(not S.lz4_frame_blocks(st)["linked"] for st in S.split_streams(seg))
        assert ("decompress_ns" in names) == (decode == "host_path" or not independent), names
    got, _ = read_back(table.schema, [(path, 0, len(data))], decode)
    assert check_read(got, vals) == vals["row"]           # partitions in order, rows in order inside a range partition


@pytest.mark.parametrize("decode", ["device_path", "host_path"])
def test_reader_reads_crafted_writer_files(tmp_path, decode):
    for name in sorted(CRAFTED)[::3] + ["literal_270", "match_ext_1", "offset_65523", "zeros_65537", "period3_131073"]:
        value = CRAFTED[name][0]
        table = pa.table({"b": to_arrow([value], "binary", bitmap=False)})
        path, data, offsets = write_single(tmp_path, table, "c")
        got, names = read_back(table.schema, [(path, 0, len(data))], decode)
        assert got["b"].to_pylist() == [value], name
        assert ("decompress_ns" in names) == (decode == "host_path")
    for size, table in tiny_tables().items():
        path, data, offsets = write_single(tmp_path, table, f"t{size}")
        got, _ = read_back(table.schema, [(path, 0, len(data))], decode)
        assert got.equals(table), size


def reference_frames(payload_groups, stats):
    """one segment per group of streams; every stream = u32 len | frame of independent 64 KB liblz4 blocks (FrameEncoder-shaped)"""
    segs = []
    for group in payload_groups:
        seg = b""
        for payload in group:
            chunks = [payload[o:o + 65536] for o in range(0, len(payload), 65536)]
            frame = S.lz4_frame([(c, pa.compress(c, codec="lz4_raw", asbytes=True)) for c in chunks])
            stream = struct.pack("<I", len(frame)) + frame
            assert S.lz4_frame_decode(S.lz4_frame_blocks(stream), stats) == payload
            seg += stream
        segs.append(seg)
    return segs


def _pattern_blob(rng):
    """runs of period 1..7 between random stretches: short overlapping matches (shared-memory ring), runs of period 1..3 longer than
    256 bytes at every output alignment, long overlapping runs of period >= 4, literals over 256 bytes and a far repeat"""
    out = bytearray()
    for i in range(120):
        out += _rng_bytes(rng, rng.randrange(1, 200))
        per = 1 + i % 7
        out += (_rng_bytes(rng, per) * 200)[:rng.randrange(8, 120) if i % 2 else rng.randrange(300, 600)]
    far = bytes(out[100:400])
    out += _rng_bytes(rng, 700) + far + _rng_bytes(rng, 50)
    return bytes(out)


def test_reader_reads_reference_shaped_frames_of_every_type():
    rng = random.Random(3)
    n = 6000
    table, vals = every_type_table(n, 0, seed=21)
    for v in (vals["utf8"], vals["binary"]):
        assert b"" in v
    # batches of 1, 7, 129, ... rows; has_nulls 1 where a NULL is present and on some columns without one
    cuts = [0, 1, 2, 9, 138, 1000, 1001, 3000, n]
    batches = []
    for a, b in zip(cuts, cuts[1:]):
        cols = [(ty, vals[name][a:b]) for name, ty in SCHEMA]
        hn = [None if ty == "null" else int(any(v is None for v in c) or rng.random() < 0.3) for ty, c in cols]
        batches.append(S.write_batch(cols, hn))
    groups = [[batches[0], b"".join(batches[1:4])], [b"".join(batches[4:6])], [batches[6], batches[7]]]
    stats = S.new_stats()
    segs = reference_frames(groups, stats)
    for decode in ("device_path", "host_path"):
        got, names = read_back(table.schema, segs, decode)
        assert check_read(got, vals) == list(range(n))
        assert ("decompress_ns" in names) == (decode == "host_path"), names


def test_reader_reads_reference_shaped_frames_at_every_decoder_branch():
    rng = random.Random(4)
    values = [_pattern_blob(rng) for _ in range(3)] + [v for v, _ in CRAFTED.values()] + [b""]
    schema = [("b", "binary"), ("row", "int64")]
    vals = {"b": values, "row": list(range(len(values)))}
    payloads = []
    for a in range(0, len(values), 4):
        cols = [("binary", values[a:a + 4]), ("int64", vals["row"][a:a + 4])]
        payloads.append(S.write_batch(cols, [0, 0]))
    stats = S.new_stats()
    segs = reference_frames([payloads[i:i + 3] for i in range(0, len(payloads), 3)], stats)
    # every branch of lz4_decompress_blocks_kernel: stored blocks, literals over 256 bytes, short overlapping matches from the ring,
    # runs of offset 1 / 2 / 3 and length >= 64 at every output alignment, overlapping runs of offset >= 4 and length >= 256,
    # disjoint copies from beyond the ring (offset > 3840)
    assert {(o, a) for o in (1, 2, 3) for a in range(4)} <= stats["small_offset_runs"], stats["small_offset_runs"]
    assert stats["max_overlap_len_off_ge4"] >= 256 and stats["far_offsets"] > 0 and stats["long_literals"] > 0
    assert stats["short_overlaps"] > 100 and stats["min_offset"] == 1
    assert any(s for seg in segs for st in S.split_streams(seg) for s, _ in S.lz4_frame_blocks(st)["blocks"])
    table = pa.table({"b": pa.array(values, pa.binary()), "row": pa.array(vals["row"], pa.int64())})
    for decode in ("device_path", "host_path"):
        got, names = read_back(table.schema, segs, decode)
        assert check_read(got, vals, schema) == vals["row"]
        assert ("decompress_ns" in names) == (decode == "host_path"), names


# -------------------------------------------------------------------------------------------- (e) IpcWriterExec
@pytest.mark.parametrize("codec", ["gpu_lz4", "zstd"])
def test_ipc_writer_every_type(codec):
    n = 20_000
    table, vals = every_type_table(n, 0, seed=5)
    sink = []

    def go():
        td = P.task_definition(P.ipc_writer(P.ffi_reader(table.schema, "in"), "consumer"))
        with runtime.Task(td, {"in": table.to_batches(max_chunksize=6000)}, ipc_consumers={"consumer": sink}) as task:
            assert list(task) == []
    with_env(dict(CODECS[codec], AURON_GPU_CHUNK_ROWS="6000"), go)
    assert len(sink) >= 4
    rows = []
    for seg in sink:
        rows += check_payload(segment_payload(seg, codec), vals)[0]
    assert rows == list(range(n))
