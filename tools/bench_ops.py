"""Per-operator throughput of the other BASELINE configs on ONE GPU, inputs resident in HBM (device resources), device
time per launch site from the library's CUDA-event timers (AURON_PROFILE=1).  These are the operator-level numbers the
north star asks for next to the config-2 bench line; they are not bench.py lines.

    python tools/bench_ops.py [join] [sort] [shuffle] [agg_lowcard] [strings] [filter_project] [scalar] [casts] [window] [generate]
                              [parquet_list] [parquet_zstd]

  join     cfg 3: store_sales (N rows: ss_sold_date_sk int32, ss_item_sk int32, ss_quantity int32) JOIN date_dim (73,049 rows:
           d_date_sk int32, d_year int32) on the date key, inner, build = date_dim
  sort     cfg 4 (one GPU's share): ORDER BY ss_item_sk over (ss_item_sk int32, ss_ticket_number int64, ss_ext_sales_price decimal(7,2))
  shuffle  cfg 4: hash repartition of the same rows on ss_item_sk into 200 partitions, compacted shuffle format to /dev/shm
  strings  md5(s), sha2(s, 256), sha2(s, 512), concat_ws('|', cast(i as string), s), md5(concat_ws(...)), lpad(s, mean, '0'),
           replace(s, 'a', 'xy'), translate(s, 'abc', 'xy') and initcap(s) over N rows of (s utf8, i int64), once with a mean string
           length of ~32 B and once with ~200 B; each projection feeds a COUNT so that one row leaves the GPU.  Reports
           compression-function calls per second next to rows/s and input GB/s.
  filter_project  cfg 1 shape on the expression VM: Project[a + 1, substr(s, 1, 4), CAST(d * 3 AS decimal(38, 2))] <-
           Filter[a > 100000 AND s LIKE 'a%'] over N rows (a int64 1 % NULL, s utf8 4-24 B, d int64), + COUNT / SUM so that one
           row leaves the GPU; the decimal output runs the 128-bit variant of vm_kernel
  scalar   months_between(t1, t2, true, 'America/New_York'), date_trunc('MONTH', t1) and greatest(g0, ..., g7) over N rows of
           (t1, t2 timestamp(us) in 1906-2096, g0..g7 int64 with 5 % NULL), each projection feeding a COUNT
  casts    CAST(f64 AS STRING), CAST(f32 AS STRING) over N random bit patterns; CAST(s AS DOUBLE) over three text shapes -- short
           ("123.45"), 17 significant digits ("0.12345678901234567") and 55-digit exact halfway points between neighbouring doubles,
           which take the exact fallback -- and CAST(s AS BOOLEAN), each over N rows and feeding a COUNT.  Reports expr_vm device time,
           rows/s and algorithmic GB/s (text bytes + offsets and fixed-width values, input once + output once; the formatted text's bytes
           are counted in an untimed pass).  Then the Filter -> Project leg three times, each time followed by the same leg of the
           built checkout at $OPS_PARENT when that is set
  window   WindowExec over N pre-sorted rows (p int32, ~1,000 rows per partition; o int64; v decimal(17,2), 5 % NULL; s utf8 8-24 B)
           in device batches of 16M rows, so the running state carries across batch edges: ROW_NUMBER, RANK, SUM(v), AVG(v), MAX(s),
           COUNT(v) partitioned by p ordered by o, + COUNT / SUM so that one row leaves the GPU
  generate LATERAL VIEW explode(split(s, ',')) + COUNT grouped by the element over N rows of 34 B strings (five 6-letter words from a
           vocabulary of 1,000, four separators), in device batches of 16M rows.  Reports the device time of the split kernels and of
           the generate gather with their algorithmic bytes, then the Filter -> Project leg, so that both come from the same run
  parquet_list  Parquet scan of N rows of list<int64> and of list<string> (0-8 elements, mean 4; 5 % NULL elements; SNAPPY; data
           page v1 and v2) -> explode -> COUNT.  Reports the device time of the level pass (pq_list_levels) next to the whole pass,
           then the config-2 fused leg (SNAPPY Parquet of N rows item / qty / date int32 -> Filter -> partial SUM / COUNT by item,
           best of 5 passes) and the Filter -> Project leg three times each, each time followed by the same leg of the built checkout
           at $OPS_PARENT when that is set
  parquet_zstd  the config-2 file (N rows item / qty / date int32, dictionary pages) written with ZSTD level 1, ZSTD level 3 and
           LZ4_RAW, its image resident in HBM (put_device_file) -> Filter -> partial SUM / COUNT by item.  Reports the device time of
           the page decompression kernels (pq_zstd, lz4_decompress) with compressed and uncompressed GB/s (the chunks' compressed and
           uncompressed sizes from the footer), then the whole pass (best of 5) three times, each time followed by the same pass of
           the built checkout at $OPS_PARENT when that is set
"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import decimal

import numpy as np
import pyarrow as pa

from auron_b200 import proto as P
from auron_b200 import runtime

os.environ["AURON_PROFILE"] = "1"
N = int(os.environ.get("OPS_ROWS", 64_000_000))
CHUNK = 16_000_000
which = sys.argv[1:] or ["join", "sort", "shuffle"]
rng = np.random.default_rng(42)


def put(resource, table):
    for b in table.to_batches(max_chunksize=CHUNK):
        runtime.put_device_batch(resource, b)


PEAK = 3350.0   # GB/s, H100 SXM data sheet HBM3 bandwidth


def run(plan, label, rows, steps=4, alg=None):
    """alg: {launch site: algorithmic bytes per pass} (inputs once + outputs once, DESIGN.md section 3)"""
    td = P.task_definition(plan)
    best = None
    for it in range(steps):
        t0 = time.perf_counter()
        with runtime.Task(td) as task:
            out_rows = 0
            for b in task:
                out_rows += b.num_rows
            m = task.metrics()
        dt = time.perf_counter() - t0
        if best is None or dt < best[0]:
            best = (dt, out_rows, m)
    dt, out_rows, m = best
    print(f"== {label}: {rows / dt / 1e6:.0f} Mrows/s end to end ({1000 * dt:.1f} ms per pass, {out_rows} rows out, result copied to the host)")
    kern = {}
    for _, op, name, v in m:
        if op == "__kernels__" and name.endswith(".device_us"):
            kern[name[:-10]] = v
    for k, v in sorted(kern.items(), key=lambda kv: -kv[1]):
        extra = ""
        if alg and alg.get(k) and v > 0:
            gbs = alg[k] / (v * 1e-6) / 1e9
            extra = f"   {alg[k] / 1e9:7.2f} GB algorithmic -> {gbs:7.0f} GB/s = {100 * gbs / PEAK:4.1f} % of {PEAK:.0f}"
        print(f"     {k:28s} {v / 1000:9.3f} ms{extra}")
    for _, op, name, v in m:
        if op != "__kernels__" and name.endswith("_ns") and v > 2e5:
            print(f"     [{op}.{name} = {v / 1e6:.2f} ms]")
    return kern


if "join" in which:
    date_lo = 2450816
    dd = pa.table({"d_date_sk": pa.array(np.arange(2415022, 2415022 + 73049, dtype=np.int32)),
                   "d_year": pa.array((1900 + np.arange(73049) // 365).astype(np.int32))})
    ss = pa.table({"ss_sold_date_sk": pa.array(rng.integers(date_lo, date_lo + 1826, N, dtype=np.int32), mask=rng.random(N) < 0.04),
                   "ss_item_sk": pa.array(rng.integers(1, 204001, N, dtype=np.int32)),
                   "ss_quantity": pa.array(rng.integers(1, 101, N, dtype=np.int32))})
    put("ss_join", ss)
    put("dd_join", dd)
    out_schema = pa.schema(list(dd.schema) + list(ss.schema))
    # the join output stays on the device: aggregate it to one row so that the measurement is the join, not a 1 GB D2H
    j = P.hash_join(out_schema, P.ffi_reader(dd.schema, "dd_join"), P.ffi_reader(ss.schema, "ss_join"),
                    [(P.col("d_date_sk"), P.col("ss_sold_date_sk"))], "INNER", "LEFT")
    plan = P.agg(j, [], [], [P.agg_expr("SUM", [P.col("ss_quantity")], pa.int64()), P.agg_expr("SUM", [P.col("d_year")], pa.int64()),
                             P.agg_expr("COUNT", [P.col("ss_item_sk")], pa.int64())], ["q", "y", "c"], ["PARTIAL"] * 3)
    matched = int(N * 0.96)
    run(plan, f"cfg3 HashJoin build=date_dim(73,049) probe={N} rows + global SUM/COUNT of the joined rows", N,
        alg={"join_probe": N * 4 + N // 8 + matched * 8,           # probe keys + validity in, (probe row, build row) pairs out
             "take": matched * 2 * 20,                              # 5 int32 output columns gathered: row bytes in + out
             "join_build": 73049 * 4 * 2})
    runtime.drop_device_resource("ss_join")
    runtime.drop_device_resource("dd_join")

if "sort" in which or "shuffle" in which:
    price = rng.integers(0, 2_000_000, N)
    # decimal(7,2) column built from unscaled integers without a Python loop
    unscaled = price.astype(np.int64)
    lo = unscaled.view(np.uint64)
    hi = np.where(unscaled < 0, np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64(0))
    buf = np.empty(2 * N, dtype=np.uint64)
    buf[0::2] = lo
    buf[1::2] = hi
    dec = pa.Array.from_buffers(pa.decimal128(7, 2), N, [None, pa.py_buffer(buf.tobytes())])
    t4 = pa.table({"ss_item_sk": pa.array(rng.integers(1, 204001, N, dtype=np.int32)),
                   "ss_ticket_number": pa.array(rng.integers(1, 240_000_000, N, dtype=np.int64)),
                   "ss_ext_sales_price": dec})
    put("t4", t4)
    if "sort" in which:
        # ORDER BY + LIMIT keeps the sort complete (all rows are ordered) but returns only the head to the host
        plan = P.sort(P.ffi_reader(t4.schema, "t4"), [P.sort_expr(P.col("ss_item_sk"))], limit=1000)
        run(plan, f"cfg4 SortExec ORDER BY ss_item_sk LIMIT 1000 over {N} rows x 28 B (top-k path)", N)
        plan = P.agg(P.sort(P.ffi_reader(t4.schema, "t4"), [P.sort_expr(P.col("ss_item_sk"))]), [], [],
                     [P.agg_expr("COUNT", [P.col("ss_item_sk")], pa.int64())], ["c"], ["PARTIAL"])
        run(plan, f"cfg4 SortExec full ORDER BY ss_item_sk over {N} rows x 28 B (+ COUNT so that only one row leaves the GPU)", N,
            alg={"radix_sort": 3 * 2 * 12 * N,                      # 18-bit key: 3 executed 8-bit passes x (u64 word + i32 row) read + write
                 "take": 2 * 28 * N})
    if "shuffle" in which:
        d = "/dev/shm/auron_ops_shuffle"
        os.makedirs(d, exist_ok=True)
        plan = P.shuffle_writer(P.ffi_reader(t4.schema, "t4"), P.hash_repartition([P.col("ss_item_sk")], 200), f"{d}/s.data", f"{d}/s.index")
        run(plan, f"cfg4 ShuffleWriterExec hash(ss_item_sk) -> 200 partitions, {N} rows x 28 B, LZ4 blocks written to /dev/shm", N, steps=3,
            alg={"murmur3_partition_ids": 8 * N, "partition_rows": 8 * N, "take": 2 * 28 * N, "serde_write": 2 * 28 * N,
                 "lz4_compress": 28 * N + os.path.getsize(d + "/s.data") if os.path.exists(d + "/s.data") else 28 * N})
        print(f"     shuffle file: {os.path.getsize(d + '/s.data') / 1e6:.0f} MB")
        # read side: IpcReaderExec over all 200 segments of the file just written (+ COUNT so that one row leaves the GPU)
        import struct
        offs = struct.unpack("<201q", open(f"{d}/s.index", "rb").read())
        blocks = [(f"{d}/s.data", offs[p], offs[p + 1] - offs[p]) for p in range(200)]
        rplan = P.agg(P.ipc_reader(t4.schema, "shuffle_in"), [], [], [P.agg_expr("COUNT", [P.col("ss_item_sk")], pa.int64()),
                                                                      P.agg_expr("SUM", [P.col("ss_ticket_number")], pa.int64())], ["c", "s"], ["PARTIAL"] * 2)
        td = P.task_definition(rplan)
        best = None
        for it in range(3):
            t0 = time.perf_counter()
            with runtime.Task(td, shuffle_blocks={"shuffle_in": list(blocks)}) as task:
                out = pa.Table.from_batches(list(task), schema=task.schema)
                m = task.metrics()
            dt = time.perf_counter() - t0
            if best is None or dt < best[0]:
                best = (dt, out, m)
        dt, out, m = best
        print(f"== cfg4 IpcReaderExec (shuffle read) of the same file: {N / dt / 1e6:.0f} Mrows/s ({1000 * dt:.1f} ms, count = {out.column(0).to_pylist()})")
        for _, op, name, v in m:
            if op != "__kernels__" and name.endswith("_ns") and v > 2e5:
                print(f"     [{op}.{name} = {v / 1e6:.2f} ms]")
    runtime.drop_device_resource("t4")

if "strings" in which:
    import subprocess

    def text_len(x):   # characters of CAST(int64 AS STRING)
        a = np.abs(x)
        return (x < 0).astype(np.int64) + 1 + sum((a >= 10 ** k).astype(np.int64) for k in range(1, 19))

    def digest_calls(lens, block, pad):   # compression-function calls: floor((len + pad) / block) + 1 per row
        return int(((lens + pad) // block + 1).sum())

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"== strings leg on: {gpu}")
    for mean in (32, 200):
        chunk = min(CHUNK, (1 << 31) // (2 * mean + 160))   # keeps every utf8 input and output of one batch below 2 GiB
        pool = rng.integers(32, 127, 1 << 20, dtype=np.uint8)
        lens_all, ws_all = [], []
        n_a = n_c = 0   # bytes 'a' and 'c' in all values: what replace and translate add and delete
        for start in range(0, N, chunk):
            n = min(chunk, N - start)
            lens = rng.integers(0, 2 * mean + 1, n).astype(np.int64)
            offs = np.zeros(n + 1, dtype=np.int32)
            np.cumsum(lens, out=offs[1:])
            data = np.resize(pool, int(offs[-1]))
            n_a += int(np.count_nonzero(data == ord("a")))
            n_c += int(np.count_nonzero(data == ord("c")))
            s_arr = pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offs), pa.py_buffer(data)])
            i_np = rng.integers(-2**62, 2**62, n, dtype=np.int64)
            runtime.put_device_batch(f"str{mean}", pa.record_batch([s_arr, pa.array(i_np)], names=["s", "i"]))
            lens_all.append(lens)
            ws_all.append(lens + 1 + text_len(i_np))
        lens = np.concatenate(lens_all)
        ws_lens = np.concatenate(ws_all)
        s_in = int(lens.sum()) + 4 * (N + 1)            # algorithmic bytes: string bytes + offsets
        ws_out = int(ws_lens.sum()) + 4 * (N + 1)
        schema = pa.schema([("s", pa.string()), ("i", pa.int64())])
        U = pa.string()
        ws = P.scalar_fn("Spark_StringConcatWs", [P.lit("|", U), P.cast(P.col("i"), U), P.col("s")], U)
        hexb = lambda w: N * w + 4 * (N + 1)   # noqa: E731
        # label, expression, {launch site: algorithmic bytes}, (digest site, compression calls)
        cases = [("md5(s)", P.scalar_fn("Spark_MD5", [P.col("s")], U), {"digest_md5": s_in + hexb(32)}, ("digest_md5", digest_calls(lens, 64, 8))),
                 ("sha2(s,256)", P.scalar_fn("Spark_Sha256", [P.col("s")], U), {"digest_sha256": s_in + hexb(64)},
                  ("digest_sha256", digest_calls(lens, 64, 8))),
                 ("sha2(s,512)", P.scalar_fn("Spark_Sha512", [P.col("s")], U), {"digest_sha512": s_in + hexb(128)},
                  ("digest_sha512", digest_calls(lens, 128, 16))),
                 ("concat_ws('|', cast(i as string), s)", ws, {"expr_vm": s_in + 8 * N + ws_out}, None),
                 ("md5(concat_ws(...))", P.scalar_fn("Spark_MD5", [ws], U), {"expr_vm": s_in + 8 * N + ws_out, "digest_md5": ws_out + hexb(32)},
                  ("digest_md5", digest_calls(ws_lens, 64, 8))),
                 # the values are ASCII, so characters are bytes: lpad to the mean length writes exactly `mean` bytes per row
                 (f"lpad(s, {mean}, '0')", P.scalar_fn("Lpad", [P.col("s"), P.lit(mean, pa.int64()), P.lit("0", U)], U),
                  {"expr_vm": s_in + hexb(mean)}, None),
                 ("replace(s, 'a', 'xy')", P.scalar_fn("Replace", [P.col("s"), P.lit("a", U), P.lit("xy", U)], U),
                  {"expr_vm": 2 * s_in + n_a}, None),
                 ("translate(s, 'abc', 'xy')", P.scalar_fn("Translate", [P.col("s"), P.lit("abc", U), P.lit("xy", U)], U),
                  {"expr_vm": 2 * s_in - n_c}, None),
                 ("initcap(s)", P.scalar_fn("Spark_InitCap", [P.col("s")], U), {"expr_vm": 2 * s_in}, None)]
        for label, expr, alg, digest in cases:
            proj = P.projection(P.ffi_reader(schema, f"str{mean}"), [expr], ["h"], [U])
            plan = P.agg(proj, [], [], [P.agg_expr("COUNT", [P.col("h")], pa.int64())], ["c"], ["PARTIAL"])
            us = run(plan, f"strings mean {mean} B: {label} over {N} rows", N, steps=3, alg=alg)
            if digest and us.get(digest[0]):
                site, calls = digest
                t = us[site] * 1e-6
                print(f"     {site}: {N / t / 1e9:.2f} G rows/s, {alg[site] / t / 1e9:.0f} GB/s algorithmic, "
                      f"{calls / t / 1e9:.2f} G compression calls/s ({calls / N:.2f} per row)")
        runtime.drop_device_resource(f"str{mean}")

def filter_project_leg():
    pool = rng.integers(97, 123, 1 << 20, dtype=np.uint8)
    for start in range(0, N, CHUNK):
        n = min(CHUNK, N - start)
        lens = rng.integers(4, 25, n)
        offs = np.zeros(n + 1, dtype=np.int32)
        np.cumsum(lens, out=offs[1:])
        s_arr = pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offs), pa.py_buffer(np.resize(pool, int(offs[-1])))])
        a = pa.array(rng.integers(0, 1_000_000, n), type=pa.int64(), mask=rng.random(n) < 0.01)
        runtime.put_device_batch("fp", pa.record_batch([a, s_arr, pa.array(rng.integers(-10**9, 10**9, n), type=pa.int64())], names=["a", "s", "d"]))
    sch = pa.schema([("a", pa.int64()), ("s", pa.string()), ("d", pa.int64())])
    flt = P.filter_(P.ffi_reader(sch, "fp"), [P.binary("Gt", P.col("a"), P.lit(100000, pa.int64())), P.like(P.col("s"), P.lit("a%", pa.string()))])
    proj = P.projection(flt, [P.binary("Plus", P.col("a"), P.lit(1, pa.int64())),
                              P.scalar_fn("Substr", [P.col("s"), P.lit(1, pa.int64()), P.lit(4, pa.int64())], pa.string()),
                              P.cast(P.binary("Multiply", P.col("d"), P.lit(3, pa.int64())), pa.decimal128(38, 2))],
                        ["a1", "s4", "dd"], [pa.int64(), pa.string(), pa.decimal128(38, 2)])
    plan = P.agg(proj, [], [], [P.agg_expr("COUNT", [P.col("s4")], pa.int64()), P.agg_expr("SUM", [P.col("a1")], pa.int64())], ["c", "x"], ["PARTIAL"] * 2)
    kern = run(plan, f"cfg1 shape Filter -> Project (decimal output) over {N} rows", N, steps=6)
    runtime.drop_device_resource("fp")
    return kern


if "filter_project" in which:
    filter_project_leg()

if "casts" in which:
    import re
    import subprocess

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"== casts leg on: {gpu}")
    U = pa.string()
    SUB = 8_000_000   # rows per batch of the text shapes: 8M rows x 55 B stay far below 2 GiB

    def text_array(mat):   # the fixed-width rows of a uint8 matrix as utf8
        n, w = mat.shape
        return pa.Array.from_buffers(U, n, [None, pa.py_buffer(np.arange(n + 1, dtype=np.int32) * w), pa.py_buffer(np.ascontiguousarray(mat).tobytes())])

    def digits(n, w):
        return rng.integers(48, 58, (n, w), dtype=np.uint8)

    # 55-digit exact halfway points between neighbouring doubles in [1, 2): (2m + 1) / 2^53 = (2m + 1) * 5^53 / 10^53
    half_pool = np.frombuffer(b"".join((lambda t: t[:1] + b"." + t[1:])(str((2 * int(m) + 1) * 5**53).encode())
                                       for m in rng.integers(2**52, 2**53, 1 << 16, dtype=np.int64)), dtype=np.uint8).reshape(-1, 55)
    bool_pool = np.frombuffer(b"true false    t    f  yes   no    1    0maybe", dtype=np.uint8).reshape(-1, 5)

    def shape(kind, n):
        if kind == "short":    # ddd.dd
            m = digits(n, 6)
            m[:, 3] = ord(".")
            return m
        if kind == "repr17":   # 0. and 17 significant digits
            m = digits(n, 19)
            m[:, 0], m[:, 1] = ord("0"), ord(".")
            m[:, 2] = rng.integers(49, 58, n, dtype=np.uint8)
            return m
        if kind == "halfway":
            return half_pool[rng.integers(0, len(half_pool), n)]
        return bool_pool[rng.integers(0, len(bool_pool), n)]

    for kind in ("short", "repr17", "halfway", "bool"):
        for start in range(0, N, SUB):
            runtime.put_device_batch(f"tx_{kind}", pa.record_batch([text_array(shape(kind, min(SUB, N - start)))], names=["s"]))
    for start in range(0, N, CHUNK):
        n = min(CHUNK, N - start)
        d = (rng.integers(0, 2**63, n, dtype=np.int64).view(np.uint64) | (rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63))).view(np.float64)
        g = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
        runtime.put_device_batch("fl", pa.record_batch([pa.array(d), pa.array(g)], names=["d", "g"]))
    fl_sch = pa.schema([("d", pa.float64()), ("g", pa.float32())])
    tx_sch = pa.schema([("s", U)])

    def text_bytes(col):   # untimed: the output text bytes of CAST(col AS STRING)
        proj = P.projection(P.ffi_reader(fl_sch, "fl"), [P.cast(P.col(col), U)], ["x"], [U])
        proj = P.projection(proj, [P.scalar_fn("OctetLength", [P.col("x")], pa.int32())], ["l"], [pa.int32()])
        plan = P.agg(proj, [], [], [P.agg_expr("SUM", [P.col("l")], pa.int64())], ["b"], ["PARTIAL"])
        with runtime.Task(P.task_definition(plan)) as task:
            return sum(b.column(0).to_pylist()[0] or 0 for b in task)

    # label, resource, schema, expression, result type, algorithmic bytes (input once + output once)
    cases = []
    for col, t, w in (("d", pa.float64(), 8), ("g", pa.float32(), 4)):
        cases.append((f"CAST({col} {t} AS STRING)", "fl", fl_sch, P.cast(P.col(col), U), U, w * N + text_bytes(col) + 4 * (N + 1)))
    for kind, width in (("short", 6), ("repr17", 19), ("halfway", 55)):
        cases.append((f"CAST(s AS DOUBLE), {kind} text ({width} B)", f"tx_{kind}", tx_sch, P.cast(P.col("s"), pa.float64()), pa.float64(),
                      (width + 4) * N + 8 * N))
    cases.append(("CAST(s AS BOOLEAN), 5 B text", "tx_bool", tx_sch, P.cast(P.col("s"), pa.bool_()), pa.bool_(), 9 * N + N // 8))
    for label, res, sch, expr, t, alg in cases:
        proj = P.projection(P.ffi_reader(sch, res), [expr], ["x"], [t])
        plan = P.agg(proj, [], [], [P.agg_expr("COUNT", [P.col("x")], pa.int64())], ["c"], ["PARTIAL"])
        us = run(plan, f"{label} over {N} rows", N, steps=3, alg={"expr_vm": alg})
        if us.get("expr_vm"):
            sec = us["expr_vm"] * 1e-6
            print(f"     expr_vm: {N / sec / 1e9:.2f} G rows/s, {alg / sec / 1e9:.0f} GB/s algorithmic")
    for r in ("fl", "tx_short", "tx_repr17", "tx_halfway", "tx_bool"):
        runtime.drop_device_resource(r)
    # the Filter -> Project leg, alternating with a built checkout of the parent when OPS_PARENT names one
    parent = os.environ.get("OPS_PARENT")
    for k in range(3):
        print(f"== Filter -> Project, this tree, pass {k + 1}: expr_vm {filter_project_leg().get('expr_vm', 0) / 1000:.3f} ms")
        if parent:
            out = subprocess.run([sys.executable, os.path.join(parent, "tools", "bench_ops.py"), "filter_project"], capture_output=True, text=True,
                                 cwd=parent, env=dict(os.environ, OPS_ROWS=str(N))).stdout
            ms = re.search(r"expr_vm\s+([0-9.]+) ms", out)
            print(f"== Filter -> Project, parent tree, pass {k + 1}: expr_vm {ms.group(1) if ms else '?'} ms")


if "scalar" in which:
    import subprocess

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"== scalar leg on: {gpu}")
    TS = pa.timestamp("us")
    names = ["t1", "t2"] + [f"g{k}" for k in range(8)]
    for start in range(0, N, CHUNK):
        n = min(CHUNK, N - start)
        ts = [pa.array(rng.integers(-2 * 10**15, 4 * 10**15, n)).cast(TS) for _ in range(2)]   # 1906 .. 2096
        gs = [pa.array(rng.integers(-2**62, 2**62, n), mask=rng.random(n) < 0.05) for _ in range(8)]
        runtime.put_device_batch("sc", pa.record_batch(ts + gs, names=names))
    sch = pa.schema([(k, TS) for k in names[:2]] + [(k, pa.int64()) for k in names[2:]])
    cases = [("months_between(t1, t2, true, 'America/New_York')",
              P.scalar_fn("Spark_MonthsBetween", [P.col("t1"), P.col("t2"), P.lit(True, pa.bool_()), P.lit("America/New_York", pa.string())], pa.float64()),
              pa.float64(), 2 * 8 * N + 8 * N),
             ("date_trunc('MONTH', t1)", P.scalar_fn("DateTrunc", [P.lit("MONTH", pa.string()), P.col("t1")], TS), TS, 8 * N + 8 * N),
             ("greatest(g0, ..., g7)", P.scalar_fn("Greatest", [P.col(f"g{k}") for k in range(8)], pa.int64()), pa.int64(), 8 * 8 * N + 8 * N)]
    for label, expr, t, alg in cases:   # algorithmic bytes: the input columns once + the output once (validity bits left out)
        proj = P.projection(P.ffi_reader(sch, "sc"), [expr], ["x"], [t])
        plan = P.agg(proj, [], [], [P.agg_expr("COUNT", [P.col("x")], pa.int64())], ["c"], ["PARTIAL"])
        run(plan, f"{label} over {N} rows", N, alg={"expr_vm": alg})
    runtime.drop_device_resource("sc")

if "window" in which:
    import subprocess

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"== window leg on: {gpu}")
    assert N % 1000 == 0
    pool = rng.integers(97, 123, 1 << 20, dtype=np.uint8)
    s_bytes = 0
    for start in range(0, N, CHUNK):
        n = min(CHUNK, N - start)
        p = (np.arange(start, start + n) // 1000).astype(np.int32)
        o = np.sort(rng.integers(0, 1000, n).reshape(-1, 1000), axis=1).reshape(-1)   # sorted inside every partition of 1,000 rows
        unscaled = rng.integers(-10**12, 10**12, n)
        buf = np.empty(2 * n, dtype=np.int64)
        buf[0::2] = unscaled
        buf[1::2] = np.where(unscaled < 0, -1, 0)
        valid = rng.random(n) >= 0.05
        v = pa.Array.from_buffers(pa.decimal128(17, 2), n, [pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()), pa.py_buffer(buf.tobytes())])
        lens = rng.integers(8, 25, n)
        offs = np.zeros(n + 1, dtype=np.int32)
        np.cumsum(lens, out=offs[1:])
        s_arr = pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offs), pa.py_buffer(np.resize(pool, int(offs[-1])))])
        s_bytes += int(offs[-1])
        runtime.put_device_batch("win", pa.record_batch([pa.array(p), pa.array(o), v, s_arr], names=["p", "o", "v", "s"]))
    sch = pa.schema([("p", pa.int32()), ("o", pa.int64()), ("v", pa.decimal128(17, 2)), ("s", pa.string())])
    I, L = pa.int32(), pa.int64()
    wex = [P.window_expr("rn", I, "ROW_NUMBER"), P.window_expr("rk", I, "RANK"), P.window_expr("sv", pa.decimal128(27, 2), "SUM", [P.col("v")]),
           P.window_expr("av", pa.decimal128(21, 6), "AVG", [P.col("v")]), P.window_expr("ms", pa.string(), "MAX", [P.col("s")]),
           P.window_expr("cv", L, "COUNT", [P.col("v")])]
    win = P.window(P.ffi_reader(sch, "win"), wex, [P.col("p")], [P.sort_expr(P.col("o"))])
    plan = P.agg(win, [], [], [P.agg_expr("COUNT", [P.col("ms")], L), P.agg_expr("SUM", [P.col("rn")], L), P.agg_expr("SUM", [P.col("rk")], L),
                               P.agg_expr("COUNT", [P.col("sv")], L), P.agg_expr("COUNT", [P.col("av")], L), P.agg_expr("SUM", [P.col("cv")], L)],
                 ["c", "rn", "rk", "sv", "av", "cv"], ["PARTIAL"] * 6)
    # algorithmic bytes per row of the segmented scans (input + output once, + the 1-byte boundary flags): four int64 scans (ROW_NUMBER,
    # RANK's row number, the COUNT and the two counts of SUM / AVG share the shape) + RANK's max, two i128 value scans, one int32 index
    # scan for MAX(s); the string gather reads and writes the bytes and offsets once
    scan_b = N * (17 * 6 + 33 * 2 + 9)
    run(plan, f"window ROW_NUMBER, RANK, SUM(dec), AVG(dec), MAX(utf8), COUNT over {N} rows in {(N + CHUNK - 1) // CHUNK} batches", N, steps=3,
        alg={"window_scan": scan_b, "take": 2 * (s_bytes + 4 * N)})
    runtime.drop_device_resource("win")

if "generate" in which:
    import subprocess

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"== generate leg on: {gpu}")
    U = pa.string()
    vocab = rng.integers(97, 123, (1000, 6), dtype=np.uint8)
    W, K = 6, 5   # word length, words per row: rows of K * W + K - 1 = 34 bytes
    row_b = K * W + K - 1
    for start in range(0, N, CHUNK):
        n = min(CHUNK, N - start)
        mat = np.full((n, row_b), ord(","), dtype=np.uint8)
        ids = rng.integers(0, 1000, (n, K))
        for k in range(K):
            mat[:, k * (W + 1):k * (W + 1) + W] = vocab[ids[:, k]]
        offs = np.arange(0, (n + 1) * row_b, row_b, dtype=np.int32)
        s_arr = pa.Array.from_buffers(U, n, [None, pa.py_buffer(offs), pa.py_buffer(mat.reshape(-1))])
        runtime.put_device_batch("gen", pa.record_batch([s_arr], names=["s"]))
    LU = pa.list_(U)
    proj = P.projection(P.ffi_reader(pa.schema([("s", U)]), "gen"), [P.scalar_fn("Spark_StringSplit", [P.col("s"), P.lit(",", U)], LU)], ["p"], [LU])
    gen = P.generate(proj, "Explode", P.col("p"), [], [("w", U, True)])
    plan = P.agg(gen, [P.col("w")], ["w"], [P.agg_expr("COUNT", [P.col("w")], pa.int64())], ["c"], ["PARTIAL"])
    with runtime.Task(P.task_definition(plan)) as task:   # every word once per row and position: the counts add up to K * N
        total = sum(sum(b.column(1).to_pylist()) for b in task)
    assert total == K * N, total
    # algorithmic bytes, inputs once + outputs once: split reads the strings and their offsets and writes the pieces (the bytes less the
    # separators), their offsets and the list offsets; the gather reads and writes the pieces with their offsets
    piece_b, pieces = K * W * N, K * N
    split_b = (row_b + 4) * N + piece_b + 4 * pieces + 4 * N
    take_b = 2 * (piece_b + 4 * pieces)
    run(plan, f"explode(split(s, ',')) -> COUNT by element over {N} rows of {row_b} B", N, steps=4,
        alg={"string_split": split_b, "take": take_b})
    runtime.drop_device_resource("gen")
    filter_project_leg()

if "parquet_list" in which:
    import subprocess
    import tempfile

    import pyarrow.parquet as pq

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"== parquet_list leg on: {gpu}")
    U = pa.string()
    lens = rng.integers(0, 9, N).astype(np.int32)
    offs = np.zeros(N + 1, dtype=np.int32)
    np.cumsum(lens, out=offs[1:])
    n_el = int(offs[-1])
    mask = rng.random(n_el) < 0.05
    vocab = np.array([f"tag{i:05d}" for i in range(10_000)], dtype=object)
    with tempfile.TemporaryDirectory() as d:
        for kind in ("int64", "string"):
            if kind == "int64":
                child = pa.array(rng.integers(-2**40, 2**40, n_el), pa.int64(), mask=mask)
            else:
                words = vocab[rng.integers(0, len(vocab), n_el)]
                child = pa.array(words, U, mask=mask)
            col = pa.ListArray.from_arrays(pa.array(offs), child)
            tab = pa.table({"l": col})
            for ver in ("1.0", "2.0"):
                path = os.path.join(d, f"{kind}_{ver}.parquet")
                pq.write_table(tab, path, compression="SNAPPY", data_page_version=ver, row_group_size=4 << 20)
                scan = P.parquet_scan(tab.schema, [(path, os.path.getsize(path))], [0])
                gen = P.generate(scan, "Explode", P.col("l"), [], [("w", tab.schema.field("l").type.value_type, True)])
                plan = P.agg(gen, [], [], [P.agg_expr("COUNT", [P.col("w")], pa.int64())], ["c"], ["PARTIAL"])
                with runtime.Task(P.task_definition(plan)) as task:
                    got = sum(sum(b.column(0).to_pylist()) for b in task)
                assert got == n_el - int(mask.sum()), got
                run(plan, f"parquet list<{kind}> v{ver} SNAPPY ({os.path.getsize(path) >> 20} MiB) -> explode -> COUNT over {N} rows, {n_el} elements", N,
                    steps=3)
                os.remove(path)
        # the config-2 fused leg, run in a fresh process from a tree's root (this one, then the parent's), the same file for both
        fused = os.path.join(d, "cfg2.parquet")
        pq.write_table(pa.table({"item": pa.array(rng.integers(1, 204001, N).astype(np.int32)),
                                 "qty": pa.array(rng.integers(1, 101, N).astype(np.int32), mask=rng.random(N) < 0.03),
                                 "date": pa.array(rng.integers(2450816, 2452642, N).astype(np.int32), mask=rng.random(N) < 0.04)}),
                       fused, compression="SNAPPY", row_group_size=8 << 20)
        leg = """
import os, sys, time
sys.path.insert(0, os.getcwd())
import pyarrow as pa
from auron_b200 import proto as P
from auron_b200 import runtime
path = sys.argv[1]
I32, I64 = pa.int32(), pa.int64()
sch = pa.schema([("item", I32), ("qty", I32), ("date", I32)])
flt = P.filter_(P.parquet_scan(sch, [(path, os.path.getsize(path))], [0, 1, 2]),
                [P.binary("GtEq", P.col("date"), P.lit(2451000, I32)), P.binary("Lt", P.col("date"), P.lit(2452000, I32))])
plan = P.agg(flt, [P.try_cast(P.col("item"), I64)], ["item"], [P.agg_expr("SUM", [P.col("qty")], I64), P.agg_expr("COUNT", [P.col("qty")], I64)],
             ["s", "c"], ["PARTIAL", "PARTIAL"])
best, fused = None, 0
for _ in range(5):
    t0 = time.perf_counter()
    with runtime.Task(P.task_definition(plan)) as task:
        rows = sum(b.num_rows for b in task)
        fused = sum(v for _, _, n, v in task.metrics() if n == "fused_batches")
    dt = time.perf_counter() - t0
    best = dt if best is None else min(best, dt)
print(f"fused_ms {1000 * best:.1f} groups {rows} fused_batches {fused}")
"""
        here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        parent = os.environ.get("OPS_PARENT")
        for k in range(3):
            for label, root in [("this tree", here)] + ([("parent tree", parent)] if parent else []):
                out = subprocess.run([sys.executable, "-c", leg, fused], capture_output=True, text=True, cwd=root).stdout.strip()
                print(f"== config-2 fused leg over {N} rows, {label}, pass {k + 1}: {out}")
    for k in range(3):
        print(f"== Filter -> Project, this tree, pass {k + 1}: expr_vm {filter_project_leg().get('expr_vm', 0) / 1000:.3f} ms")
        if parent:
            import re
            out = subprocess.run([sys.executable, os.path.join(parent, "tools", "bench_ops.py"), "filter_project"], capture_output=True, text=True,
                                 cwd=parent, env=dict(os.environ, OPS_ROWS=str(N))).stdout
            ms = re.search(r"expr_vm\s+([0-9.]+) ms", out)
            print(f"== Filter -> Project, parent tree, pass {k + 1}: expr_vm {ms.group(1) if ms else '?'} ms")

if "parquet_zstd" in which:
    import subprocess
    import tempfile

    import pyarrow.parquet as pq

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"== parquet_zstd leg on: {gpu}")
    tab = pa.table({"item": pa.array(rng.integers(1, 204001, N).astype(np.int32)),
                    "qty": pa.array(rng.integers(1, 101, N).astype(np.int32), mask=rng.random(N) < 0.03),
                    "date": pa.array(rng.integers(2450816, 2452642, N).astype(np.int32), mask=rng.random(N) < 0.04)})
    leg = """
import os, sys, time
sys.path.insert(0, os.getcwd())
import pyarrow as pa
from auron_b200 import proto as P
from auron_b200 import runtime
path = sys.argv[1]
data = open(path, "rb").read()
runtime.put_device_file("hbm://cfg2", data)
I32, I64 = pa.int32(), pa.int64()
sch = pa.schema([("item", I32), ("qty", I32), ("date", I32)])
flt = P.filter_(P.parquet_scan(sch, [("hbm://cfg2", len(data))], [0, 1, 2]),
                [P.binary("GtEq", P.col("date"), P.lit(2451000, I32)), P.binary("Lt", P.col("date"), P.lit(2452000, I32))])
plan = P.agg(flt, [P.try_cast(P.col("item"), I64)], ["item"], [P.agg_expr("SUM", [P.col("qty")], I64), P.agg_expr("COUNT", [P.col("qty")], I64)],
             ["s", "c"], ["PARTIAL", "PARTIAL"])
best, fused, total = None, 0, 0
for _ in range(5):
    t0 = time.perf_counter()
    with runtime.Task(P.task_definition(plan)) as task:
        rows, tot = 0, 0
        for b in task:
            rows += b.num_rows
            tot += sum(x for x in b.column(2).to_pylist() if x)
        fused = sum(v for _, _, n, v in task.metrics() if n == "fused_batches")
    dt = time.perf_counter() - t0
    best = dt if best is None else min(best, dt)
print(f"pass_ms {1000 * best:.1f} groups {rows} count {tot} fused_batches {fused}")
"""
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    parent = os.environ.get("OPS_PARENT")
    with tempfile.TemporaryDirectory() as d:
        for codec, level in (("ZSTD", 1), ("ZSTD", 3), ("LZ4_RAW", None)):
            path = os.path.join(d, f"cfg2_{codec}_{level}.parquet")
            pq.write_table(tab, path, compression=codec, row_group_size=8 << 20, **({"compression_level": level} if level else {}))
            md = pq.ParquetFile(path).metadata
            comp = sum(md.row_group(g).column(c).total_compressed_size for g in range(md.num_row_groups) for c in range(md.num_columns))
            unc = sum(md.row_group(g).column(c).total_uncompressed_size for g in range(md.num_row_groups) for c in range(md.num_columns))
            name = f"{codec}" + (f" level {level}" if level else "")
            data = open(path, "rb").read()
            runtime.put_device_file("hbm://zs", data)
            sch = tab.schema
            flt = P.filter_(P.parquet_scan(sch, [("hbm://zs", len(data))], [0, 1, 2]),
                            [P.binary("GtEq", P.col("date"), P.lit(2451000, pa.int32())), P.binary("Lt", P.col("date"), P.lit(2452000, pa.int32()))])
            plan = P.agg(flt, [P.try_cast(P.col("item"), pa.int64())], ["item"],
                         [P.agg_expr("SUM", [P.col("qty")], pa.int64()), P.agg_expr("COUNT", [P.col("qty")], pa.int64())], ["s", "c"], ["PARTIAL", "PARTIAL"])
            kern = run(plan, f"config-2 {name} image in HBM ({comp >> 20} MiB compressed, {unc >> 20} MiB uncompressed) -> Filter -> SUM / COUNT by item over {N} rows",
                       N, steps=3)
            for site in ("pq_zstd", "lz4_decompress"):
                if kern.get(site):
                    sec = kern[site] * 1e-6
                    print(f"     {site}: {comp / sec / 1e9:.1f} GB/s compressed in, {unc / sec / 1e9:.1f} GB/s uncompressed out, "
                          f"{(comp + unc) / sec / 1e9:.1f} GB/s algorithmic")
            runtime.drop_device_file("hbm://zs")
            for k in range(3):
                for label, root in [("this tree", here)] + ([("parent tree", parent)] if parent else []):
                    out = subprocess.run([sys.executable, "-c", leg, path], capture_output=True, text=True, cwd=root)
                    print(f"== config-2 {name} pass over {N} rows, {label}, round {k + 1}: {out.stdout.strip() or out.stderr.strip()[-300:]}")
