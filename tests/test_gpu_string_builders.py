"""md5 / sha2 digests and the string constructors (concat, concat_ws, repeat, space) on the GPU, against the reference's golden
tables and a Python restatement of its semantics (paths relative to native-engine/datafusion-ext-functions/src):
  * Spark_MD5 / Spark_Sha224/256/384/512: lowercase hex digest of a utf8 or binary value's bytes, NULL -> NULL (spark_crypto.rs:33-105)
  * Spark_StringConcat: NULL if any argument is NULL (spark_strings.rs:117-192)
  * Spark_StringConcatWs: literal separator; NULL arguments are skipped with their separator; never NULL otherwise (:194-319)
  * Spark_StringRepeat: literal int32 count; NULL count -> every row NULL, n < 0 -> "", NULL string -> NULL (:75-91)
  * Spark_StringSpace: NULL -> NULL, n < 0 -> "" (:65-73)
"""
import datetime as dt
import decimal
import hashlib

import numpy as np
import pyarrow as pa
import pytest

import oracle
from auron_b200 import proto as P
from helpers import assert_same_rows, run
from test_gpu_shuffle import read_shuffle_files

pytestmark = pytest.mark.gpu

U = pa.string()
DIGESTS = {"Spark_MD5": hashlib.md5, "Spark_Sha224": hashlib.sha224, "Spark_Sha256": hashlib.sha256, "Spark_Sha384": hashlib.sha384,
           "Spark_Sha512": hashlib.sha512}


def fn(name, *args):
    return P.scalar_fn(name, list(args), U)


def lit(v, t=U):
    return P.lit(v, t)


def project(t, exprs, rid="t", src=None):
    src = src or P.ffi_reader(t.schema, rid)
    return P.projection(src, exprs, [f"c{i}" for i in range(len(exprs))], [U] * len(exprs))


def column(t, expr, **kw):
    return run(project(t, [expr]), {"t": t}, **kw).column(0).to_pylist()


# ---------------------------------------------------------------------------------------------- Python restatement
def py_digest(name, v):
    if v is None:
        return None
    return DIGESTS[name](v.encode() if isinstance(v, str) else v).hexdigest()


def py_concat(*vals):
    return None if any(v is None for v in vals) else "".join(vals)


def py_concat_ws(sep, *vals):
    return sep.join(v for v in vals if v is not None)


def py_upper(v):   # the VM's upper() is ASCII-only
    return None if v is None else "".join(chr(ord(c) - 32) if "a" <= c <= "z" else c for c in v)


def py_dec(v):
    return None if v is None else format(v, "f")


# ---------------------------------------------------------------------------------------------- reference goldens
def test_crypto_goldens_utf8_and_binary():
    # spark_crypto.rs:140-208
    exp = {"Spark_MD5": ("902fbdd2b1df0c4f70b4a5d23525e932", "6ac1e56bc78f031059be7be854522c4c"),
           "Spark_Sha224": ("107c5072b799c4771f328304cfe1ebb375eb6ea7f35a3aa753836fad", "4225cbc32d17010d1a440de9e34504c1fae29b8ee5e527e191ff9a82"),
           "Spark_Sha256": ("b5d4045c3f466fa91fe2cc6abe79232a1a57cdf104f7a26e716e0a1e2789df78",
                            "7192385c3c0605de55bb9476ce1d90748190ecb32a8eed7f5207b30cf6a1fe89"),
           "Spark_Sha384": ("1e02dc92a41db610c9bcdc9b5935d1fb9be5639116f6c67e97bc1a3ac649753baba7ba021c813e1fe20c0480213ad371",
                            "557cfe660c753b830efa61528fc350ef384a7a4b9d3467c6230049bc59548eb8a404874baff89cb0f9bd18400829fdc2"),
           "Spark_Sha512": ("397118fdac8d83ad98813c50759c85b8c47565d8268bf10da483153b747a74743a58a90e85aa9f705ce6984ffc128db567489817e4092d050d8a1cc596ddc119",
                            "178d767c364244ede054ebb3cc4af0ac2b307a86fba6a32706ce4f692642674d2ab8f51ee738ecb09bc296918aa85db48abe28fcaef7aa2da81a618cc6d891c3")}
    t = pa.table({"s": pa.array(["ABC", None]), "b": pa.array([bytes([1, 2, 3, 4, 5, 6]), None], type=pa.binary())})
    out = run(project(t, [fn(n, P.col(c)) for n in exp for c in ("s", "b")]), {"t": t})
    for k, n in enumerate(exp):
        assert out.column(2 * k).to_pylist() == [exp[n][0], None], n
        assert out.column(2 * k + 1).to_pylist() == [exp[n][1], None], n
        assert out.schema.field(2 * k).type == U


def test_space_golden():
    # spark_strings.rs:340-353
    t = pa.table({"n": pa.array([3, 0, -100, None], type=pa.int32())})
    assert column(t, fn("Spark_StringSpace", P.col("n"))) == ["   ", "", "", None]


def test_repeat_goldens():
    # spark_strings.rs:398-445: n = 3, n < 0, n = NULL
    t = pa.table({"s": pa.array(["123", "a", None])})
    assert column(t, fn("Spark_StringRepeat", P.col("s"), lit(3, pa.int32()))) == ["123123123", "aaa", None]
    assert column(t, fn("Spark_StringRepeat", P.col("s"), lit(-1, pa.int32()))) == ["", "", None]
    assert column(t, fn("Spark_StringRepeat", P.col("s"), lit(None, pa.int32()))) == [None, None, None]


def test_concat_golden():
    # spark_strings.rs:482-506
    t = pa.table({"a": pa.array(["123", None]), "b": pa.array(["444", "456"]), "c": pa.array(["", ""])})
    assert column(t, fn("Spark_StringConcat", P.col("a"), P.col("b"), P.col("c"), lit("SomeScalar"))) == ["123444SomeScalar", None]


def test_concat_ws_golden_without_the_list_argument():
    # spark_strings.rs:507-541 with its array<string> argument left out (nested types are not built)
    t = pa.table({"a": pa.array(["123", None]), "b": pa.array([None, "456"]), "c": pa.array(["", ""])})
    e = fn("Spark_StringConcatWs", lit("||"), P.col("a"), P.col("b"), P.col("c"), lit("SomeScalar"), lit(None))
    assert column(t, e) == ["123||||SomeScalar", "456||||SomeScalar"]
    assert column(t, fn("Spark_StringConcatWs", lit(None), P.col("a"))) == [None, None]


# ---------------------------------------------------------------------------------------------- fuzz
def _fuzz_table(n, seed):
    rng = np.random.default_rng(seed)
    pool = "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyzABCXYZ 0123456789|-éßж天地😁"), 4096))
    null = lambda: rng.random(n) < 0.05   # noqa: E731
    starts, lens = rng.integers(0, 3000, n), rng.integers(0, 301, n)
    s = [pool[a:a + k] for a, k in zip(starts, lens)]
    b = [rng.bytes(int(k)) for k in rng.integers(0, 301, n)]   # binary with NUL bytes
    words = ["", "x", "ab", "Mixed Case", "天地"]
    return pa.table({
        "s": pa.array(s, mask=null()),
        "b": pa.array(b, type=pa.binary(), mask=null()),
        "w": pa.array([words[int(k)] for k in rng.integers(0, len(words), n)], mask=null()),
        "i": pa.array(rng.integers(-2**62, 2**62, n), type=pa.int64(), mask=null()),
        "n": pa.array(rng.integers(-5, 40, n), type=pa.int32(), mask=null()),
        "k": pa.array(rng.integers(0, 100, n), type=pa.int32()),
    })


def _fuzz_exprs():
    return [fn("Spark_MD5", P.col("s")), fn("Spark_Sha224", P.col("s")), fn("Spark_Sha256", P.col("b")), fn("Spark_Sha384", P.col("s")),
            fn("Spark_Sha512", P.col("b")), fn("Spark_MD5", P.col("b")),
            fn("Spark_StringConcat", P.col("w"), lit("-"), fn("Upper", P.col("s"))),
            fn("Spark_StringConcatWs", lit("|"), P.col("w"), P.cast(P.col("i"), U), P.col("s")),
            fn("Spark_StringRepeat", P.col("w"), lit(2, pa.int32())),
            fn("Spark_StringSpace", P.col("n")),
            fn("Spark_Sha256", fn("Spark_StringConcatWs", lit("|"), P.col("w"), P.col("s")))]


def _fuzz_expected(t):
    c = {k: t.column(k).to_pylist() for k in t.column_names}
    rows = list(zip(c["s"], c["b"], c["w"], c["i"], c["n"]))
    cols = [[py_digest("Spark_MD5", s) for s, *_ in rows], [py_digest("Spark_Sha224", s) for s, *_ in rows],
            [py_digest("Spark_Sha256", b) for _, b, *_ in rows], [py_digest("Spark_Sha384", s) for s, *_ in rows],
            [py_digest("Spark_Sha512", b) for _, b, *_ in rows], [py_digest("Spark_MD5", b) for _, b, *_ in rows],
            [py_concat(w, "-", py_upper(s)) for s, _, w, _, _ in rows],
            [py_concat_ws("|", w, None if i is None else str(i), s) for s, _, w, i, _ in rows],
            [None if w is None else w * 2 for _, _, w, _, _ in rows],
            [None if n is None else " " * max(n, 0) for *_, n in rows],
            [py_digest("Spark_Sha256", py_concat_ws("|", w, s)) for s, _, w, _, _ in rows]]
    return pa.table({f"c{k}": pa.array(v, type=U) for k, v in enumerate(cols)})


def test_fuzz_against_hashlib_several_batches():
    t = _fuzz_table(200_000, seed=11)
    got = run(project(t, _fuzz_exprs()), {"t": t}, chunk=70_000)
    exp = _fuzz_expected(t)
    for k in range(exp.num_columns):
        assert got.column(k).to_pylist() == exp.column(k).to_pylist(), k


def test_fuzz_below_a_filter_and_with_no_rows_selected():
    t = _fuzz_table(60_000, seed=12)
    flt = P.filter_(P.ffi_reader(t.schema, "t"), [P.binary("Lt", P.col("k"), P.lit(37, pa.int32()))])   # sel is non-null
    got = run(project(t, _fuzz_exprs(), src=flt), {"t": t}, chunk=25_000)
    exp = _fuzz_expected(t.filter(pa.array(np.asarray(t.column("k")) < 37)))
    for k in range(exp.num_columns):
        assert got.column(k).to_pylist() == exp.column(k).to_pylist(), k
    # a Filter that keeps no row of a non-empty batch: the projection, its hidden digest arguments included, runs over zero rows
    none = P.filter_(P.ffi_reader(t.schema, "t"), [P.binary("Lt", P.col("k"), P.lit(0, pa.int32()))])
    empty = run(project(t, _fuzz_exprs(), src=none), {"t": t}, chunk=25_000)
    assert empty.num_rows == 0 and empty.num_columns == len(_fuzz_exprs())
    assert all(f.type == U for f in empty.schema)


def test_row_fingerprint():
    rng = np.random.default_rng(5)
    n = 50_000
    words = ["alpha", "Beta", "", "天地", None]
    t = pa.table({"i": pa.array(rng.integers(-2**63, 2**63 - 1, n), type=pa.int64(), mask=rng.random(n) < 0.05),
                  "s": pa.array([words[int(k)] for k in rng.integers(0, len(words), n)]),
                  "d": pa.array(rng.integers(-800_000, 2_900_000, n).astype(np.int32), type=pa.date32(), mask=rng.random(n) < 0.05),
                  "m": pa.array([None if x else decimal.Decimal(int(v)).scaleb(-2) for x, v in zip(rng.random(n) < 0.05, rng.integers(-10**16, 10**16, n))],
                                type=pa.decimal128(17, 2))})
    pieces = [P.cast(P.col("i"), U), P.col("s"), P.cast(P.col("d"), U), P.cast(P.col("m"), U), fn("Upper", P.col("s"))]
    out = run(project(t, [fn("Spark_MD5", fn("Spark_StringConcatWs", lit("|"), *pieces)),
                          fn("Spark_Sha256", fn("Spark_StringConcat", *pieces))]), {"t": t}, chunk=20_000)
    # the device's date text is the proleptic Gregorian yyyy-mm-dd with at least four year digits
    days = t.column("d").cast(pa.int32()).to_pylist()

    def date_text(v):
        if v is None:
            return None
        y, m, d = _civil(v)
        return ("-" if y < 0 else "") + f"{abs(y):04d}-{m:02d}-{d:02d}"

    rows = zip(t.column("i").to_pylist(), t.column("s").to_pylist(), days, t.column("m").to_pylist())
    exp_md5, exp_sha = [], []
    for i, s, d, m in rows:
        vals = [None if i is None else str(i), s, date_text(d), py_dec(m), py_upper(s)]
        exp_md5.append(py_digest("Spark_MD5", py_concat_ws("|", *vals)))
        exp_sha.append(py_digest("Spark_Sha256", py_concat(*vals)))
    assert out.column(0).to_pylist() == exp_md5
    assert out.column(1).to_pylist() == exp_sha


def _civil(z):   # days since 1970-01-01 -> (year, month, day), proleptic Gregorian for any year
    z += 719468
    era = z // 146097   # floor division, as the device's (z - 146096) / 146097 for negative z
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = mp + 3 if mp < 10 else mp - 9
    return yoe + era * 400 + (m <= 2), m, d


def test_date_text_helper_matches_python_dates():
    for v in (-719162, -1, 0, 59, 10957, 2932896):
        y, m, d = _civil(v)
        assert dt.date(1970, 1, 1) + dt.timedelta(days=v) == dt.date(y, m, d)


def test_long_values():
    rng = np.random.default_rng(9)
    vals = [rng.bytes(64 << 10), rng.bytes(1 << 20), None, rng.bytes((1 << 20) + 37), rng.bytes((64 << 10) - 1), b""]
    t = pa.table({"b": pa.array(vals, type=pa.binary())})
    out = run(project(t, [fn(n, P.col("b")) for n in DIGESTS]), {"t": t})
    for k, n in enumerate(DIGESTS):
        assert out.column(k).to_pylist() == [py_digest(n, v) for v in vals], n
    s = pa.table({"s": pa.array(["ab" * (32 << 10), None, "x"])})
    assert column(s, fn("Spark_StringRepeat", P.col("s"), lit(16, pa.int32()))) == ["ab" * (512 << 10), None, "x" * 16]


# ---------------------------------------------------------------------------------------------- query level
def test_group_by_md5_partial_and_final():
    rng = np.random.default_rng(21)
    n = 120_000
    t = pa.table({"s": pa.array([f"key-{int(k)}" for k in rng.integers(0, 500, n)], mask=rng.random(n) < 0.02),
                  "v": pa.array(rng.integers(0, 10, n), type=pa.int64())})
    key = fn("Spark_MD5", fn("Spark_StringConcatWs", lit("|"), P.col("s"), lit("salt")))
    partial = P.agg(P.ffi_reader(t.schema, "t"), [key], ["h"], [P.agg_expr("COUNT", [P.col("v")], pa.int64())], ["c"], ["PARTIAL"])
    final = P.agg(partial, [P.col("h")], ["h"], [P.agg_expr("COUNT", [P.lit(None, pa.null())], pa.int64())], ["c"], ["FINAL"])
    got = run(final, {"t": t}, chunk=40_000)
    counts = {}
    for s in t.column("s").to_pylist():
        h = py_digest("Spark_MD5", py_concat_ws("|", s, "salt"))
        counts[h] = counts.get(h, 0) + 1
    assert_same_rows(got, pa.table({"h": pa.array(list(counts), type=U), "c": pa.array(list(counts.values()), type=pa.int64())}))


def test_hash_shuffle_partitioned_on_concat(tmp_path):
    rng = np.random.default_rng(31)
    n, nparts = 80_000, 16
    t = pa.table({"a": pa.array([f"a{int(k)}" for k in rng.integers(0, 3000, n)], mask=rng.random(n) < 0.03),
                  "b": pa.array([f"b{int(k)}" for k in rng.integers(0, 70, n)]),
                  "x": pa.array(np.arange(n), type=pa.int64())})
    data, index = str(tmp_path / "c.data"), str(tmp_path / "c.index")
    run(P.shuffle_writer(P.ffi_reader(t.schema, "t"), P.hash_repartition([fn("Spark_StringConcat", P.col("a"), P.col("b"))], nparts), data, index),
        {"t": t}, chunk=30_000)
    parts, _ = read_shuffle_files(data, index, t.schema)
    key = pa.array([py_concat(a, b) for a, b in zip(t.column("a").to_pylist(), t.column("b").to_pylist())], type=U)
    pid = oracle.partition_ids([key], nparts)
    for p in range(nparts):
        assert_same_rows(parts[p], t.filter(pa.array(pid == p)))
    assert sum(x.num_rows for x in parts) == n


def test_tpcds_q5_style_store_id():
    # q5 / q80: 'store' || s_store_id (Spark Concat)
    t = pa.table({"s_store_id": pa.array(["AAAAAAAABAAAAAAA", "AAAAAAAACAAAAAAA", None]), "sales": pa.array([1, 2, 3], type=pa.int64())})
    plan = P.projection(P.ffi_reader(t.schema, "t"), [fn("Spark_StringConcat", lit("store"), P.col("s_store_id")), P.col("sales")],
                        ["id", "sales"], [U, pa.int64()])
    got = run(plan, {"t": t})
    assert got.column(0).to_pylist() == ["storeAAAAAAAABAAAAAAA", "storeAAAAAAAACAAAAAAA", None]
    assert got.column(1).to_pylist() == [1, 2, 3]
