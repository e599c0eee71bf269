"""Sort, grouping, join and partition keys at the edges of every key type, against the plain-Python references of
key_reference.py.  Each operator turns key values into something else before it works (order-preserving sort words, 64-bit
hash-table keys with a sentinel, direct-address slots, i128 sums in two atomics, murmur3 partition ids); a mistake in any of
those mappings gives a wrong order or wrong groups without an error, so every case compares values exactly.  Edge values
are placed on both sides of the 2048-row scan blocks and 4096-row radix tiles (key_reference.edge_column)."""
import os
import struct

import numpy as np
import pyarrow as pa
import pytest

import key_reference as R
import oracle
from auron_b200 import proto as P
from auron_b200 import runtime
from helpers import batches
from test_gpu_ops import _join
from test_gpu_shuffle import read_shuffle_files

pytestmark = pytest.mark.gpu

ARROW = {"int8": pa.int8(), "int16": pa.int16(), "int32": pa.int32(), "int64": pa.int64(), "float32": pa.float32(), "float64": pa.float64(),
         "bool": pa.bool_(), "date32": pa.date32(), "date64": pa.date64(), "ts_s": pa.timestamp("s"), "ts_ms": pa.timestamp("ms"),
         "ts_us": pa.timestamp("us"), "ts_ns": pa.timestamp("ns"), "dec9_2": pa.decimal128(9, 2), "dec18_0": pa.decimal128(18, 0),
         "dec38_10": pa.decimal128(38, 10), "utf8": pa.string(), "binary": pa.binary()}
NUMPY = {"int8": np.int8, "int16": np.int16, "int32": np.int32, "int64": np.int64, "float32": np.uint32, "float64": np.uint64,
         "date32": np.int32, "date64": np.int64, "ts_s": np.int64, "ts_ms": np.int64, "ts_us": np.int64, "ts_ns": np.int64}
MASK128 = (1 << 128) - 1
BITMAPS = ["nulls", "no_nulls_with_bitmap", "no_bitmap"]


# -------------------------------------------------------------------------------------------- canonical values <-> Arrow
def to_arrow(vals, t, bitmap=True):
    """canonical values -> Arrow array; bitmap: keep a validity bitmap even when no value is NULL"""
    n = len(vals)
    valid = np.array([v is not None for v in vals], dtype=bool)
    vbuf = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()) if (bitmap or not valid.all()) else None
    if t == "bool":
        bufs = [vbuf, pa.py_buffer(np.packbits(np.array([bool(v) for v in vals]), bitorder="little").tobytes())]
    elif t in R.DECIMALS:
        bufs = [vbuf, pa.py_buffer(b"".join(((v or 0) & MASK128).to_bytes(16, "little") for v in vals))]
    elif t in ("utf8", "binary"):
        a = pa.array([b"" if v is None else v for v in vals], type=pa.binary())
        bufs = [vbuf, a.buffers()[1], a.buffers()[2]]
    else:
        bufs = [vbuf, pa.py_buffer(np.array([v or 0 for v in vals], dtype=NUMPY[t]).tobytes())]
    # null_count -1 (not computed yet): pyarrow drops a bitmap whose null count is given as 0
    return pa.Array.from_buffers(ARROW[t], n, bufs, null_count=-1 if vbuf is not None else 0)


def from_arrow(arr, t):
    """Arrow array (any offset) -> canonical values: floats as bits, decimals unscaled, dates / timestamps as ints"""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    n, off = len(arr), arr.offset
    if t == "bool":
        vals = arr.to_pylist()
    elif t in ("utf8", "binary"):
        vals = arr.cast(pa.binary()).to_pylist()
    elif t in R.DECIMALS:
        raw = arr.buffers()[1].to_pybytes()[off * 16:(off + n) * 16]
        vals = [int.from_bytes(raw[16 * i:16 * i + 16], "little", signed=True) for i in range(n)]
    else:
        vals = np.frombuffer(arr.buffers()[1], dtype=NUMPY[t])[off:off + n].tolist()
    valid = arr.is_valid().to_pylist()
    return [v if ok else None for v, ok in zip(vals, valid)]


def column(t, n, seed, bitmap="nulls", rate=0.2):
    vals = R.edge_column(t, n, seed, rate=rate, null_rate=0.05 if bitmap == "nulls" else 0.0)
    return vals, to_arrow(vals, t, bitmap != "no_bitmap")


def table_of(cols: dict) -> pa.Table:
    """{name: (values, arrow array)} -> table, plus a `row` payload column"""
    n = len(next(iter(cols.values()))[0])
    return pa.table({**{k: a for k, (_, a) in cols.items()}, "row": pa.array(np.arange(n), type=pa.int64())})


def run_plan(plan, inputs, env=None, chunk=None):
    env = env or {}
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        with runtime.Task(P.task_definition(plan), {k: batches(v, chunk) for k, v in inputs.items()}) as task:
            got = pa.Table.from_batches(list(task), schema=task.schema)
            met = {(op, name): v for _, op, name, v in task.metrics()}
        return got, met
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# -------------------------------------------------------------------------------------------- sort (S1, k_sort.cu)
def check_sort(t, cols, specs, env=None, chunk=None, limit=None, offset=0):
    """sort `t` by [(name, type, asc, nulls_first)]: the key sequence must equal the reference's order exactly, and every row must
    appear once with its own key values (the `row` payload)"""
    plan = P.sort(P.ffi_reader(t.schema, "t"), [P.sort_expr(P.col(c), a, nf) for c, _, a, nf in specs], limit=limit, offset=offset)
    got, met = run_plan(plan, {"t": t}, env, chunk)
    n = t.num_rows
    rows_in = list(zip(*[cols[c] for c, _, _, _ in specs]))
    rspecs = [(ty, a, nf) for _, ty, a, nf in specs]
    exp = sorted(rows_in, key=lambda r: R.row_sort_key(r, rspecs))
    hi = n if limit is None else min(n, limit)
    exp = exp[offset:hi]
    got_keys = list(zip(*[from_arrow(got[c], ty) for c, ty, _, _ in specs]))
    assert len(got_keys) == len(exp)
    bad = [i for i, (g, e) in enumerate(zip(got_keys, exp)) if g != e]
    assert not bad, (specs, bad[:3], [(got_keys[i], exp[i]) for i in bad[:3]])
    got_rows = got["row"].to_pylist()
    assert all(rows_in[r] == k for r, k in zip(got_rows, got_keys))
    if limit is None and offset == 0:
        assert sorted(got_rows) == list(range(n))
    return met


@pytest.mark.parametrize("t", R.TYPES)
def test_sort_one_key_every_direction(t):
    for bi, bitmap in enumerate(BITMAPS):
        vals, arr = column(t, 10_000 + bi, seed=11 + bi, bitmap=bitmap)
        tab = table_of({"k": (vals, arr)})
        for asc in (True, False):
            for nf in (True, False):
                check_sort(tab, {"k": vals}, [("k", t, asc, nf)], chunk=3_000)


MULTI = [(("int8", True, True), ("int64", False, False)), (("bool", False, False), ("dec38_10", True, True)),
         (("date32", True, False), ("utf8", False, True)), (("int8", False, True), ("binary", True, False)),
         (("bool", True, True), ("float64", False, True)), (("date32", False, False), ("dec38_10", False, True))]


@pytest.mark.parametrize("narrow,wide", MULTI)
def test_sort_folded_narrow_key_with_wide_key(narrow, wide):
    (tn, an, nfn), (tw, aw, nfw) = narrow, wide
    vn, a1 = column(tn, 9_000, seed=3, rate=0.6)
    vw, a2 = column(tw, 9_000, seed=4, rate=0.6)
    tab = table_of({"a": (vn, a1), "b": (vw, a2)})
    check_sort(tab, {"a": vn, "b": vw}, [("a", tn, an, nfn), ("b", tw, aw, nfw)])
    check_sort(tab, {"a": vn, "b": vw}, [("b", tw, not aw, nfw), ("a", tn, an, not nfn)])


@pytest.mark.parametrize("spill", [False, True])
def test_external_sort_every_fixed_width_type(spill):
    env = {"AURON_SORT_RUN_ROWS": "3000", **({"AURON_SORT_SPILL_BYTES": "1"} if spill else {})}
    for i, t in enumerate(R.FIXED_WIDTH):
        vals, arr = column(t, 14_000, seed=40 + i, bitmap=BITMAPS[i % 3])
        tab = table_of({"k": (vals, arr)})
        asc, nf = bool(i & 1), bool(i & 2)
        met = check_sort(tab, {"k": vals}, [("k", t, asc, nf)], env=env, chunk=5_000)
        assert met[("SortExec", "sorted_runs")] >= 4, met
        assert (met.get(("SortExec", "mem_spill_count"), 0) > 0) == spill
    vals, arr = column("dec38_10", 14_000, seed=77)
    check_sort(table_of({"k": (vals, arr)}), {"k": vals}, [("k", "dec38_10", False, False)], env=env, chunk=5_000, limit=9_000, offset=1_234)


@pytest.mark.parametrize("case", ["nine_int64", "six_decimal38", "eight_int64_one_int32"])
def test_external_sort_past_sixteen_key_words(case):
    # a sort key word per NULL rank plus one per int64 (two per decimal128): these keys need 17-18 words per row, which the run
    # splitters must compare across several runs
    types = {"nine_int64": ["int64"] * 9, "six_decimal38": ["dec38_10"] * 6, "eight_int64_one_int32": ["int64"] * 8 + ["int32"]}[case]
    cols, arrs = {}, {}
    for i, t in enumerate(types):
        vals, arr = column(t, 12_000, seed=90 + i, rate=0.9)          # few distinct values: ties reach the last key
        cols[f"k{i}"], arrs[f"k{i}"] = vals, (vals, arr)
    tab = table_of(arrs)
    specs = [(f"k{i}", t, i % 2 == 0, i % 3 == 0) for i, t in enumerate(types)]
    met = check_sort(tab, cols, specs, env={"AURON_SORT_RUN_ROWS": "2500"}, chunk=4_000)
    assert met[("SortExec", "sorted_runs")] >= 4, met


def test_sort_merge_join_past_sixteen_key_words():
    # six nullable decimal(38) keys: 18 words, compared when each side is cut into key-disjoint pieces (a join takes at most
    # eight key columns)
    lvals = {f"k{i}": R.edge_column("dec38_10", 4_000, seed=200 + i, rate=0.97, null_rate=0.01) for i in range(6)}
    # the right side repeats some left key tuples so that the join has matches
    rvals = {k: v[:1_500] + R.edge_column("dec38_10", 1_500, seed=300 + i, rate=0.97, null_rate=0.01) for i, (k, v) in enumerate(lvals.items())}
    lt = table_of({k: (v, to_arrow(v, "dec38_10")) for k, v in lvals.items()}).rename_columns([*lvals, "lrow"])
    rt = table_of({k: (v, to_arrow(v, "dec38_10")) for k, v in rvals.items()}).rename_columns([*rvals, "rrow"])
    on = [(k, k) for k in lvals]
    lk, rk = list(zip(*lvals.values())), list(zip(*rvals.values()))
    for jt in ("INNER", "LEFT", "ANTI"):
        got = _join(lt, rt, on, jt, "smj", chunk=1_000)
        check_pairs(got, R.join_rows(lk, rk, jt), jt)


# -------------------------------------------------------------------------------------------- hash aggregate (A1-A4, k_agg.cu)
AGG_PATHS = {"direct": {"AURON_FORCE_DIRECT_AGG": "1"}, "fast": {"AURON_DISABLE_DIRECT_AGG": "1"}, "general": {}, "nokey": {}}
DIRECT_TYPES = ("int8", "int16", "int32", "int64", "date32")


def agg_two_stage(tab, keys, aggs, env, chunk=4_000):
    """PARTIAL -> FINAL over device chunks of `chunk` rows; aggs = [(fn, column, return type)]"""
    names = [f"a{i}" for i in range(len(aggs))]
    src = P.ffi_reader(tab.schema, "t")
    part = P.agg(src, [P.col(k) for k in keys], keys, [P.agg_expr(f, [P.col(c)], rt) for f, c, rt in aggs], names, ["PARTIAL"] * len(aggs))
    final = P.agg(part, [P.col(k) for k in keys], keys, [P.agg_expr(f, [P.lit(None, pa.null())], rt) for f, _, rt in aggs], names,
                  ["FINAL"] * len(aggs))
    got, _ = run_plan(final, {"t": tab}, {"AURON_GPU_CHUNK_ROWS": str(chunk), **env}, chunk=chunk)
    return got


def grouped(got, key_types, out_types):
    nk = len(key_types)
    keys = list(zip(*[from_arrow(got.column(i), t) for i, t in enumerate(key_types)])) if nk else [()] * got.num_rows
    vals = list(zip(*[from_arrow(got.column(nk + j), t) for j, t in enumerate(out_types)]))
    d = dict(zip(keys, vals))
    assert len(d) == got.num_rows, "a group was emitted twice"
    return d


@pytest.mark.parametrize("t,path", [(t, p) for t in R.TYPES for p in AGG_PATHS if p != "direct" or t in DIRECT_TYPES])   # direct: integer keys only
def test_group_by_every_key_type_on_every_table_path(t, path):
    for bi, bitmap in enumerate(BITMAPS):
        n = 13_000 + bi
        kv, ka = column(t, n, seed=500 + bi, bitmap=bitmap, rate=0.5)
        rng = np.random.default_rng(bi)
        v = [int(x) for x in rng.integers(-2**63, 2**63, n)]
        g2 = [i % 3 for i in range(n)]
        tab = table_of({"k": (kv, ka), "g": (g2, to_arrow(g2, "int32")), "v": (v, to_arrow(v, "int64"))})
        keys, ktypes = {"direct": (["k"], [t]), "fast": (["k"], [t]), "general": (["k", "g"], [t, "int32"]), "nokey": ([], [])}[path]
        aggs = [("SUM", "v", pa.int64()), ("COUNT", "v", pa.int64()), ("MIN", "row", pa.int64()), ("MAX", "row", pa.int64())]
        got = grouped(agg_two_stage(tab, keys, aggs, AGG_PATHS[path]), ktypes, ["int64"] * 4)
        cols = {"k": kv, "g": g2}
        exp = {}
        for key, rows in R.group_rows(list(zip(*[cols[k] for k in keys])) if keys else [()] * n).items():
            exp[key] = (R.wrapping_sum([v[r] for r in rows]), len(rows), min(rows), max(rows))
        assert got == exp, (t, path, bitmap, len(got), len(exp))


@pytest.mark.parametrize("t", ["int8", "int16", "int32", "int64", "date32", "float32", "float64"])
def test_group_by_shared_memory_variant(t):
    # the per-CTA shared-memory pre-aggregation runs on chunks of at least 2^20 rows whose sample has few groups: the edge values
    # only (plus NULL), tiled 64 times
    base, _ = column(t, 1 << 14, seed=61, rate=0.95)
    kv = base * 64
    n = len(kv)
    rng = np.random.default_rng(5)
    vbase = [int(x) for x in rng.integers(-2**62, 2**62, 1 << 14)]
    tab = pa.table({"k": to_arrow(kv, t), "v": to_arrow(vbase * 64, "int64")})
    aggs = [("SUM", "v", pa.int64()), ("COUNT", "v", pa.int64()), ("MIN", "v", pa.int64()), ("MAX", "v", pa.int64())]
    got = grouped(agg_two_stage(tab, ["k"], aggs, {"AURON_ENABLE_SMEM_AGG": "1"}, chunk=n), [t], ["int64"] * 4)
    exp = {}
    for key, rows in R.group_rows([(k,) for k in base]).items():
        vs = [vbase[r] for r in rows]
        exp[key] = (R.wrapping_sum(vs * 64), 64 * len(vs), min(vs), max(vs))
    assert got == exp


@pytest.mark.parametrize("t,lo", [("int64", -2**63), ("int64", 2**63 - 101), ("int32", -2**31), ("int32", 2**31 - 101),
                                  ("int16", -2**15), ("int16", 2**15 - 101), ("int8", -128), ("int8", 27), ("date32", -2**31)])
@pytest.mark.parametrize("path", ["direct", "fast", "general"])
def test_group_by_keys_at_the_ends_of_the_integer_range(t, lo, path):
    rng = np.random.default_rng(lo & 0xffff)
    n = 40_000
    kv = [None if x < 0.03 else lo + int(d) for x, d in zip(rng.random(n), rng.integers(0, 101, n))]
    v = [int(x) for x in rng.integers(-10**6, 10**6, n)]
    g = [0] * n
    tab = table_of({"k": (kv, to_arrow(kv, t)), "g": (g, to_arrow(g, "int32")), "v": (v, to_arrow(v, "int64"))})
    keys, ktypes = (["k", "g"], [t, "int32"]) if path == "general" else (["k"], [t])
    got = grouped(agg_two_stage(tab, keys, [("SUM", "v", pa.int64()), ("COUNT", "v", pa.int64())], AGG_PATHS[path], chunk=15_000),
                  ktypes, ["int64", "int64"])
    exp = {(k + ((0,) if path == "general" else ())): (R.wrapping_sum([v[r] for r in rows]), len(rows))
           for k, rows in R.group_rows([(k,) for k in kv]).items()}
    assert got == exp


@pytest.mark.parametrize("with_nulls", [False, True])
@pytest.mark.parametrize("t,sentinel", [("int64", R.SENTINEL_I64), ("float64", R.SENTINEL)])
def test_group_by_the_hash_table_sentinel(t, sentinel, with_nulls):
    rng = np.random.default_rng(8)
    n = 20_000
    others = [x for x in R.edge_values(t) if x != sentinel][:4]
    kv = [sentinel if u < 0.4 else (None if with_nulls and u < 0.5 else others[int(u * 100) % 4]) for u in rng.random(n)]
    v = [int(x) for x in rng.integers(-1000, 1000, n)]
    tab = table_of({"k": (kv, to_arrow(kv, t, with_nulls)), "v": (v, to_arrow(v, "int64"))})
    exp = {k: (R.wrapping_sum([v[r] for r in rows]), len(rows)) for k, rows in R.group_rows([(k,) for k in kv]).items()}
    for path in ("fast", "direct", "general"):
        keys = ["k"] if path != "general" else ["k", "k"]
        got = grouped(agg_two_stage(tab, keys, [("SUM", "v", pa.int64()), ("COUNT", "v", pa.int64())], AGG_PATHS[path]),
                      [t] * len(keys), ["int64", "int64"])
        assert {k[:1]: s for k, s in got.items()} == exp, path


@pytest.mark.parametrize("t", ["int8", "int16", "int32", "int64"])
def test_integer_sums_wrap(t):
    n = 12_000
    vals, arr = column(t, n, seed=12, rate=0.9)
    hi = (1 << (R.INT_BITS[t] - 1)) - 1
    vals[:2], vals[-2:] = [hi, hi], [hi, hi]                           # 2 x max in one group and in another chunk
    arr = to_arrow(vals, t)
    k = [i % 5 for i in range(n)]
    tab = table_of({"k": (k, to_arrow(k, "int32")), "v": (vals, arr)})
    for keys in (["k"], []):
        got = grouped(agg_two_stage(tab, keys, [("SUM", "v", pa.int64())], {}), ["int32"] * len(keys), ["int64"])
        exp = {key: (R.wrapping_sum([vals[r] for r in rows]),) for key, rows in R.group_rows([tuple(k[i] for _ in keys) for i in range(n)]).items()}
        assert got == exp, keys


def test_decimal38_sum_and_avg_carry_both_ways_across_chunks():
    rng = np.random.default_rng(38)
    n = 16_000
    edges = R.edge_values("dec38_10")
    vals = []
    for i in range(n):
        u = rng.random()
        if u < 0.03:
            vals.append(None)
        elif u < 0.15:
            vals.append(edges[i % len(edges)])
        else:                                                          # near +-10^37: the low word carries up and borrows down
            vals.append((1 if u < 0.58 else -1) * (10 ** 37 - int(rng.integers(0, 2**63)) * 3))
    k = [i % 4 for i in range(n)]
    tab = table_of({"k": (k, to_arrow(k, "int32")), "v": (vals, to_arrow(vals, "dec38_10"))})
    d = pa.decimal128(38, 10)
    for keys in (["k"], []):
        got = grouped(agg_two_stage(tab, keys, [("SUM", "v", d), ("AVG", "v", d)], {}), ["int32"] * len(keys), ["dec38_10", "dec38_10"])
        exp = {}
        for key, rows in R.group_rows([tuple(k[i] for _ in keys) for i in range(n)]).items():
            vs = [vals[r] for r in rows]
            exp[key] = (R.wrapping_sum(vs, 128), R.decimal_avg(vs))
        assert got == exp, keys


MINMAX_TYPES = ["int8", "int16", "int32", "int64", "float32", "float64", "date32", "date64", "ts_s", "ts_ms", "ts_us", "ts_ns",
                "dec9_2", "dec18_0"]


@pytest.mark.parametrize("t", MINMAX_TYPES)
def test_min_max_of_every_fixed_width_type_in_total_order(t):
    n = 12_000
    vals, arr = column(t, n, seed=71, rate=0.7)
    k = [i % 7 for i in range(n)]
    vals = [None if kk == 6 and i < n // 2 else x for i, (kk, x) in enumerate(zip(k, vals))]   # group 6: NULL in the first chunks
    tab = table_of({"k": (k, to_arrow(k, "int32")), "v": (vals, to_arrow(vals, t))})
    at = ARROW[t]
    for keys in (["k"], []):
        got = grouped(agg_two_stage(tab, keys, [("MIN", "v", at), ("MAX", "v", at)], {}), ["int32"] * len(keys), [t, t])
        exp = {}
        for key, rows in R.group_rows([tuple(k[i] for _ in keys) for i in range(n)]).items():
            vs = [vals[r] for r in rows]
            exp[key] = (R.extreme(vs, t, False), R.extreme(vs, t, True))
        assert got == exp, keys


@pytest.mark.parametrize("t,message", [("dec38_10", "MIN/MAX over decimal"), ("bool", r"MIN/MAX\(bool\)")])
def test_min_max_of_unsupported_types_fails_naming_the_type(t, message):
    # MIN / MAX over decimals beyond 18 digits and over booleans are not on the device: an error naming the type, never a value
    vals = R.edge_values(t)
    tab = pa.table({"k": pa.array([1] * len(vals), type=pa.int32()), "v": to_arrow(vals, t)})
    for fn in ("MIN", "MAX"):
        plan = P.agg(P.ffi_reader(tab.schema, "t"), [P.col("k")], ["k"], [P.agg_expr(fn, [P.col("v")], ARROW[t])], ["m"], ["PARTIAL"])
        with pytest.raises(runtime.AuronError, match=message) as e:
            run_plan(plan, {"t": tab})
        assert t != "dec38_10" or "38" in str(e.value)


# -------------------------------------------------------------------------------------------- joins (J1-J4, k_join.cu)
JOIN_TYPES = ["INNER", "LEFT", "RIGHT", "FULL", "SEMI", "ANTI"]


def check_pairs(got, exp, jt):
    lr = got["l_lrow"].to_pylist()
    rr = got["r_rrow"].to_pylist() if jt not in ("SEMI", "ANTI") else [None] * len(lr)
    pairs = sorted(zip(lr, rr), key=lambda p: (p[0] is None, p[0] or 0, p[1] is None, p[1] or 0))
    assert pairs == exp, (jt, len(pairs), len(exp), [p for p in pairs if p not in set(exp)][:5])


def join_tables(lvals, rvals, t, lbitmap=True, rbitmap=True):
    lt = pa.table({"k": to_arrow(lvals, t, lbitmap), "lrow": pa.array(np.arange(len(lvals)), type=pa.int64())})
    rt = pa.table({"k": to_arrow(rvals, t, rbitmap), "rrow": pa.array(np.arange(len(rvals)), type=pa.int64())})
    return lt, rt


def check_join(lvals, rvals, t, impls=("shjR", "bhjL"), env=None, chunk=None):
    lt, rt = join_tables(lvals, rvals, t)
    for impl in impls:
        for jt in JOIN_TYPES:
            got = with_env(env or {}, lambda: _join(lt, rt, [("k", "k")], jt, impl, chunk=chunk))
            check_pairs(got, R.join_rows([(v,) for v in lvals], [(v,) for v in rvals], jt), jt)


@pytest.mark.parametrize("t", R.TYPES)
def test_join_on_every_key_type_with_duplicates(t):
    # floats match by their bits: NaN meets NaN of the same payload, -0.0 does not meet +0.0 (DESIGN section 4)
    lvals = R.edge_column(t, 3_000, seed=31, rate=0.3)
    rvals = R.edge_column(t, 2_000, seed=32, rate=0.3) + lvals[:50]
    check_join(lvals, rvals, t, impls=("shjR", "bhjL", "smj"), chunk=1_000)


@pytest.mark.parametrize("t", DIRECT_TYPES)
@pytest.mark.parametrize("end", ["min", "max"])
@pytest.mark.parametrize("mask", [True, False])
def test_join_direct_table_at_the_ends_of_the_key_range(t, end, mask):
    # unique build keys in a small range take the direct-address table (slot = key - dmin, compared unsigned against the range);
    # probe keys just outside it, far outside it and at the opposite extreme make key - dmin wrap
    bits = 32 if t == "date32" else R.INT_BITS[t]
    tmin, tmax = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    span = 60
    lo = tmin if end == "min" else tmax - span + 1
    build = list(range(lo, lo + span))
    near = [x for x in (lo - 1, lo + span, lo - 2, lo + span + 1) if tmin <= x <= tmax]
    probe = build + near + [tmin, tmax, 0, -1, tmin + 1, tmax - 1, None] * 3
    probe = probe * 20
    env = {} if mask else {"AURON_JOIN_NO_MASK": "1"}
    # the build side: right for shjR, left for bhjL
    lt, rt = join_tables(probe, build, t)
    for jt in JOIN_TYPES:
        with_env(env, lambda: check_pairs(_join(lt, rt, [("k", "k")], jt, "shjR"), R.join_rows([(v,) for v in probe], [(v,) for v in build], jt), jt))
    lt, rt = join_tables(build, probe, t)
    for jt in JOIN_TYPES:
        with_env(env, lambda: check_pairs(_join(lt, rt, [("k", "k")], jt, "bhjL"), R.join_rows([(v,) for v in build], [(v,) for v in probe], jt), jt))
    for jt in ("INNER", "LEFT", "FULL"):
        check_pairs(_join(lt, rt, [("k", "k")], jt, "smj"), R.join_rows([(v,) for v in build], [(v,) for v in probe], jt), jt)


def with_env(env, fn):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return fn()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def test_join_unique_keys_over_the_whole_int64_range():
    rng = np.random.default_rng(64)
    build = sorted(set(int(x) for x in rng.integers(-2**63, 2**63, 5_000)) | set(R.edge_values("int64")))
    probe = [build[int(i)] if u < 0.6 else int(x) for u, i, x in zip(rng.random(20_000), rng.integers(0, len(build), 20_000),
                                                                       rng.integers(-2**63, 2**63, 20_000))]
    probe += [None] * 100
    for mask in (True, False):
        with_env({} if mask else {"AURON_JOIN_NO_MASK": "1"}, lambda: check_join(probe, build, "int64", impls=("shjR",)))
    check_join(build, probe, "int64", impls=("bhjL", "smj"))


@pytest.mark.parametrize("t,sentinel", [("int64", R.SENTINEL_I64), ("float64", R.SENTINEL)])
def test_join_on_the_hash_table_sentinel(t, sentinel):
    others = [x for x in R.edge_values(t) if x != sentinel]
    for lvals, rvals in ([others * 3, others + [sentinel]],                       # build side only
                         [others + [sentinel] * 4, others * 2],                   # probe side only
                         [others + [sentinel] * 3 + [None], [sentinel, sentinel] + others]):   # both
        check_join(lvals, rvals, t, impls=("shjR", "bhjL", "smj"))
        check_join(lvals, rvals, t, impls=("shjR", "bhjL"), env={"AURON_JOIN_NO_MASK": "1"})


def test_join_general_path_on_decimal_high_words_and_multi_keys():
    w = 1 << 64
    dl = [1, 1 + w, 1 - w, 1 + 2 * w, 5, None, -(w - 1), 10 ** 38 - 1] * 40
    dr = [1 + w, 1 - w, 1, 7, None, -(w - 1), -(10 ** 38 - 1)] * 30
    check_join(dl, dr, "dec38_10", impls=("shjR", "bhjL", "smj"))
    # bool + binary + float64 as one key (row-key path)
    n = 2_500
    cl = {"b": R.edge_column("bool", n, 1, rate=0.5), "s": R.edge_column("binary", n, 2, rate=0.9), "f": R.edge_column("float64", n, 3, rate=0.9)}
    cr = {c: v[:800] + R.edge_column(t, 800, 9, rate=0.9) for (c, v), t in zip(cl.items(), ("bool", "binary", "float64"))}
    types = {"b": "bool", "s": "binary", "f": "float64"}
    lt = pa.table({**{c: to_arrow(v, types[c]) for c, v in cl.items()}, "lrow": pa.array(np.arange(n), type=pa.int64())})
    rt = pa.table({**{c: to_arrow(v, types[c]) for c, v in cr.items()}, "rrow": pa.array(np.arange(1600), type=pa.int64())})
    lk, rk = list(zip(*cl.values())), list(zip(*cr.values()))
    for impl in ("shjR", "bhjL"):
        for jt in JOIN_TYPES:
            check_pairs(_join(lt, rt, [(c, c) for c in cl], jt, impl), R.join_rows(lk, rk, jt), jt)


# -------------------------------------------------------------------------------------------- partitioning (S2-S4, k_hash.cu)
DIVISORS = [1, 2, 3, 7, 8191, 8192, 8193, 65537, 2**31 - 1]


@pytest.mark.parametrize("t", R.TYPES)
def test_partition_ids_of_every_type_and_divisor(t):
    for r in range(4):                                                # n % 4 = 0, 1, 2, 3: the 4-rows-per-thread kernel's tail
        vals, arr = column(t, 10_000 + r, seed=80 + r, bitmap=BITMAPS[r % 3])
        vals2, arr2 = column("int32", 10_000 + r, seed=90 + r)
        b = pa.record_batch({"k": arr, "j": arr2})
        for cols in ([0], [0, 1]):
            for d in DIVISORS:
                got = runtime.k_partition_ids(b, cols, d).to_numpy()
                exp = oracle.partition_ids([b.column(c) for c in cols], d)
                assert (got == exp).all(), (t, r, cols, d)
                rows = with_env({"AURON_DISABLE_HASH_FIXED4": "1"}, lambda: runtime.k_partition_ids(b, cols, d).to_numpy())
                assert (rows == got).all(), (t, r, cols, d)


def test_hash_shuffle_write_with_more_partitions_than_the_shared_histogram(tmp_path):
    # 8193 partitions: pid_hist_kernel counts with global atomics instead of shared memory
    nparts = 8193
    kv, ka = column("int64", 60_000, seed=13)
    sv, sa = column("utf8", 60_000, seed=14)
    t = table_of({"k": (kv, ka), "s": (sv, sa)})
    data, index = str(tmp_path / "p.data"), str(tmp_path / "p.index")
    plan = P.shuffle_writer(P.ffi_reader(t.schema, "t"), P.hash_repartition([P.col("k"), P.col("s")], nparts), data, index)
    run_plan(plan, {"t": t}, chunk=25_000)
    parts, offsets = read_shuffle_files(data, index, t.schema)
    assert len(offsets) == nparts + 1
    pid = oracle.partition_ids([t["k"].combine_chunks(), t["s"].combine_chunks()], nparts)
    got = {}
    for p in range(nparts):
        for r in parts[p]["row"].to_pylist():
            got[r] = p
    assert len(got) == t.num_rows
    assert all(got[r] == pid[r] for r in range(t.num_rows))
    rows = {r: (k, s) for r, k, s in zip(range(t.num_rows), kv, sv)}
    for p in range(0, nparts, 97):                                     # payload travelled with its row
        part = parts[p]
        assert [rows[r] for r in part["row"].to_pylist()] == list(zip(from_arrow(part["k"], "int64"), from_arrow(part["s"], "utf8")))


def _bound_values(t, vals):
    if t == "float64":
        return [struct.unpack("<d", struct.pack("<Q", v))[0] for v in vals]
    if t == "dec38_10":
        return [R.unscaled_to_decimal(v, 10) for v in vals]
    return [v.decode() for v in vals]


@pytest.mark.parametrize("t,asc,nf", [("float64", True, True), ("float64", False, False), ("dec38_10", True, False), ("dec38_10", False, True),
                                      ("utf8", True, True), ("utf8", False, False)])
def test_range_partition_bounds_equal_to_keys(tmp_path, t, asc, nf):
    # partition = number of bounds strictly below the key in sort order (bisect_left); bounds are edge values, so keys equal them
    edges = {"float64": [R.f64_bits(x) for x in (float("-inf"), -0.0, 0.0, 1.0, float("nan"))],
             "dec38_10": [-(10 ** 38 - 1), -(1 << 64), 1 - (1 << 64), 0, 1, 1 << 64, 10 ** 38 - 1],
             "utf8": [b"", b"a", b"a\x00", b"q" * 15 + b"b", "é".encode(), "\U0001F600".encode()]}[t]
    bounds = sorted(edges, key=lambda v: R.sort_key(v, t, asc, nf))
    vals, arr = column(t, 20_000, seed=21)
    tab = table_of({"k": (vals, arr)})
    nparts = len(bounds) + 1
    data, index = str(tmp_path / "r.data"), str(tmp_path / "r.index")
    plan = P.shuffle_writer(P.ffi_reader(tab.schema, "t"), P.range_repartition([P.sort_expr(P.col("k"), asc, nf)], nparts,
                                                                               [(_bound_values(t, bounds), ARROW[t])]), data, index)
    run_plan(plan, {"t": tab}, chunk=7_000)
    parts, _ = read_shuffle_files(data, index, tab.schema)
    got = {}
    for p in range(nparts):
        for r in parts[p]["row"].to_pylist():
            got[r] = p
    exp = R.range_partition_ids([(v,) for v in vals], [(b,) for b in bounds], [(t, asc, nf)])
    assert [got[r] for r in range(len(vals))] == exp
