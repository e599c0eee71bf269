"""CAST(utf8 AS FLOAT / DOUBLE / BOOLEAN) and CAST(float / double / decimal(38, s) AS STRING) on the GPU, row by row against the
plain-Python reference in cast_reference.py (its docstring states the semantics), with NULLs, every special and malformed form,
over several batches, below a Filter, and in the positions the planner accepts them."""
import decimal
import hashlib
import random
import struct

import numpy as np
import pyarrow as pa
import pytest

import cast_reference as R
from auron_b200 import proto as P
from helpers import run

pytestmark = pytest.mark.gpu
EXACT = decimal.Context(prec=80)

U, F32, F64, BOOL, I64 = pa.string(), pa.float32(), pa.float64(), pa.bool_(), pa.int64()
SPECIALS = ["+NaN", "nan", "NAN", "INF", "+nan", "-Infinity", "Infinity", "-inf", "+infinity", "1.5d", "1.5F", "1e400", "-1e-400",
            "\t 2.5 \n", ".5", "5.", "", ".", "e5", "1e", "1.5 d", "1_0", "0x1.8p1", "١", "1e+", "--1", "123", "321.9", "-098", "sda",
            "2.2250738585072011e-308", "2.4703282292062327e-324", "2.4703282292062328e-324", "1.7976931348623158e308",
            "1.7976931348623159e308", "9007199254740993", "7.038531e-26", "1" * 40 + "e-20", "0." + "0" * 30 + "1",
            "t", "TRUE", " yes\t", "no", "0", "1", "F", "on"]


def _texts(n, seed):
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        r = rng.random()
        if r < 0.05:
            out.append(None)
        elif r < 0.25:
            out.append(rng.choice(SPECIALS))
        elif r < 0.5:
            out.append(repr(struct.unpack("<d", struct.pack("<Q", rng.getrandbits(63)))[0]))
        elif r < 0.65:
            out.append("".join(rng.choice("0123456789") for _ in range(rng.randint(20, 40))) + "e" + str(rng.randint(-340, 300)))
        else:
            out.append("%.*g" % (rng.randint(1, 9), rng.uniform(-1e6, 1e6)))
    return out


def _bits_col(col, bits):
    fmt = "<d" if bits == 64 else "<f"
    return [None if v is None else struct.unpack("<Q" if bits == 64 else "<I", struct.pack(fmt, v))[0] for v in col.to_pylist()]


def _canon_nan(bits_list, bits):
    nan = R.NAN[bits]
    mb = 52 if bits == 64 else 23
    full = (1 << bits) - 1
    out = []
    for b in bits_list:
        if b is not None and ((b & (full >> 1)) >> mb) == (1 << (bits - 1 - mb)) - 1 and b & ((1 << mb) - 1):
            b = nan
        out.append(b)
    return out


def check(got, exp, what):
    assert len(got) == len(exp), what
    bad = [i for i, (a, b) in enumerate(zip(got, exp)) if a != b]
    assert not bad, (what, len(bad), [(i, got[i], exp[i]) for i in bad[:4]])


@pytest.mark.parametrize("try_cast,filtered", [(False, False), (True, True)])
def test_text_to_float_and_bool_fuzz(try_cast, filtered):
    texts = _texts(200_000, 1)
    keep = [i % 3 != 1 for i in range(len(texts))]
    t = pa.table({"s": pa.array(texts, U), "k": pa.array(np.arange(len(texts)), I64), "keep": pa.array(keep, BOOL)})
    c = P.try_cast if try_cast else P.cast
    src = P.ffi_reader(t.schema, "t")
    if filtered:
        src = P.filter_(src, [P.col("keep")])
        texts = [s for s, k in zip(texts, keep) if k]
    plan = P.projection(src, [P.col("k"), c(P.col("s"), F64), c(P.col("s"), F32), c(P.col("s"), BOOL),
                              c(P.scalar_fn("Trim", [P.col("s")], U), F64)],
                        ["k", "d", "f", "b", "td"], [I64, F64, F32, BOOL, F64])
    out = run(plan, {"t": t}, chunk=70_000).sort_by("k")
    assert out.num_rows == len(texts)
    check(_canon_nan(_bits_col(out.column("d"), 64), 64), [R.to_float(s, 64) for s in texts], "double")
    check(_canon_nan(_bits_col(out.column("f"), 32), 32), [R.to_float(s, 32) for s in texts], "float")
    check(out.column("b").to_pylist(), [R.to_bool(s) for s in texts], "bool")
    check(_canon_nan(_bits_col(out.column("td"), 64), 64), [R.to_float(None if s is None else s.strip(" "), 64) for s in texts], "trim")


def test_float_to_text_fuzz_below_a_filter():
    rng = random.Random(2)
    n = 200_000
    pats = [rng.getrandbits(64) if i % 5 else rng.getrandbits(52) for i in range(n)]
    d = [struct.unpack("<d", struct.pack("<Q", b))[0] for b in pats]
    f32 = np.array([rng.getrandbits(32) for _ in range(n)], dtype=np.uint32).view(np.float32)
    keep = [i % 3 != 0 for i in range(n)]
    t = pa.table({"d": pa.array(d, F64, mask=np.array([i % 17 == 0 for i in range(n)])), "g": pa.array(f32, F32),
                  "k": pa.array(np.arange(n), I64), "keep": pa.array(keep, BOOL)})
    src = P.filter_(P.ffi_reader(t.schema, "t"), [P.col("keep")])
    plan = P.projection(src, [P.col("k"), P.cast(P.col("d"), U), P.try_cast(P.col("g"), U)], ["k", "ds", "gs"], [I64, U, U])
    out = run(plan, {"t": t}, chunk=60_000).sort_by("k")
    ks = out.column("k").to_pylist()
    assert ks == [i for i in range(n) if keep[i]]
    check(out.column("ds").to_pylist(), [None if i % 17 == 0 else R.float_to_text(pats[i], 64) for i in ks], "double")
    gb = f32.view(np.uint32)
    check(out.column("gs").to_pylist(), [R.float_to_text(int(gb[i]), 32) for i in ks], "float")


def test_java_goldens_on_the_device():
    doubles = [(0.1 + 0.2, "0.30000000000000004"), (1e23, "1.0E23"), (5e-324, "4.9E-324"), (1e-323, "9.9E-324"),
               (2.2250738585072014e-308, "2.2250738585072014E-308"), (9999999.0, "9999999.0"), (1.23456789e7, "1.23456789E7"),
               (0.001, "0.001"), (1e7, "1.0E7"), (1e-4, "1.0E-4"), (1.7976931348623157e308, "1.7976931348623157E308"), (-0.0, "-0.0"),
               (float("inf"), "Infinity"), (float("-inf"), "-Infinity"), (float("nan"), "NaN")]
    floats = [(3.4028234663852886e38, "3.4028235E38"), (16777216.0, "1.6777216E7"), (1.401298464324817e-45, "1.4E-45"), (0.1, "0.1")]
    floats += [(0.0, "0.0")] * (len(doubles) - len(floats))
    t = pa.table({"d": pa.array([x for x, _ in doubles], F64), "g": pa.array([x for x, _ in floats], F32)})
    out = run(P.projection(P.ffi_reader(t.schema, "t"), [P.cast(P.col("d"), U), P.cast(P.col("g"), U)], ["a", "b"], [U, U]), {"t": t})
    assert out.column("a").to_pylist() == [s for _, s in doubles]
    assert out.column("b").to_pylist() == [s for _, s in floats]
    texts = {"+NaN": "NaN", "INF": "Infinity", "+nan": None, "1.5d": "1.5", "1e400": "Infinity", "-1e-400": "-0.0", "0x1.8p1": None}
    t = pa.table({"s": pa.array(list(texts), U)})
    out = run(P.projection(P.ffi_reader(t.schema, "t"), [P.cast(P.cast(P.col("s"), F64), U)], ["a"], [U]), {"t": t})
    assert out.column("a").to_pylist() == list(texts.values())


def test_hash_shuffle_keys(tmp_path):
    from test_gpu_shuffle import read_shuffle_files

    import oracle
    texts = _texts(30_000, 7)
    rng = np.random.default_rng(8)
    d = rng.integers(0, 2**63, len(texts), dtype=np.int64).view(np.float64)
    t = pa.table({"s": pa.array(texts, U), "d": pa.array(d, F64), "x": pa.array(np.arange(len(texts)), I64)})
    ref_d = [None if b is None else struct.unpack("<d", struct.pack("<Q", b))[0] for b in _canon_nan([R.to_float(s, 64) for s in texts], 64)]
    ref_s = [R.float_to_text(struct.unpack("<Q", struct.pack("<d", v))[0], 64) for v in d]
    for name, key, keys in (("double", P.try_cast(P.col("s"), F64), pa.array(ref_d, F64)), ("text", P.cast(P.col("d"), U), pa.array(ref_s, U))):
        data, index = str(tmp_path / f"{name}.data"), str(tmp_path / f"{name}.index")
        run(P.shuffle_writer(P.ffi_reader(t.schema, "t"), P.hash_repartition([key], 8), data, index), {"t": t}, chunk=10_000)
        parts, _ = read_shuffle_files(data, index, t.schema)
        pid = oracle.partition_ids([keys], 8)
        for p in range(8):
            assert sorted(parts[p].column("x").to_pylist()) == [i for i in range(len(texts)) if pid[i] == p], (name, p)


def test_decimal38_to_text_at_the_edges():
    for s in (0, 1, 18, 37, 38):
        vals = [10**38 - 1, -(10**38 - 1), 0, 1, -1, 2**64, -(2**64) - 1, 123 * 10**18, None]
        arr = pa.array([None if v is None else decimal.Decimal(v).scaleb(-s, EXACT) for v in vals], pa.decimal128(38, s))
        t = pa.table({"x": arr})
        plan = P.projection(P.ffi_reader(t.schema, "t"), [P.cast(P.col("x"), U),
                                                          P.scalar_fn("Spark_StringConcat", [P.lit("<", U), P.cast(P.col("x"), U)], U)],
                            ["a", "b"], [U, U])
        out = run(plan, {"t": t})
        exp = [R.decimal_to_text(v, s) for v in vals]
        check(out.column("a").to_pylist(), exp, s)
        check(out.column("b").to_pylist(), [None if e is None else "<" + e for e in exp], s)


def test_casts_in_every_position():
    texts = ["1.5", "2.5", "x", None, "t", "no", "-3", "1e3"] * 500
    n = len(texts)
    dec = pa.array([decimal.Decimal(i % 7).scaleb(-10, EXACT) for i in range(n)], pa.decimal128(38, 10))
    dv = [float(i % 5) / 4 for i in range(n)]
    t = pa.table({"s": pa.array(texts, U), "d": pa.array(dv, F64), "m": dec, "k": pa.array(np.arange(n), I64)})
    src = lambda: P.ffi_reader(t.schema, "t")   # noqa: E731
    to_d = P.try_cast(P.col("s"), F64)
    ref_d = [None if R.to_float(s, 64) is None else struct.unpack("<d", struct.pack("<Q", R.to_float(s, 64)))[0] for s in texts]
    # Filter predicate
    out = run(P.projection(P.filter_(src(), [P.binary("Gt", to_d, P.lit(1.0, F64))]), [P.col("k")], ["k"], [I64]), {"t": t})
    assert sorted(out.column(0).to_pylist()) == [i for i, v in enumerate(ref_d) if v is not None and v > 1.0]
    # SUM(CAST(s AS DOUBLE)) and GROUP BY CAST(s AS BOOLEAN)
    out = run(P.agg(src(), [P.cast(P.col("s"), BOOL)], ["b"], [P.agg_expr("SUM", [to_d], F64)], ["x"], ["PARTIAL"]), {"t": t})
    got = dict(zip(out.column(0).to_pylist(), out.column(1).to_pylist()))
    for key in (True, False, None):
        vals = [v for s, v in zip(texts, ref_d) if R.to_bool(s) is key and v is not None]
        assert (got.get(key) or 0.0) == pytest.approx(sum(vals)), key
    # CASE branch
    case = P.case([(P.binary("Eq", P.col("s"), P.lit("x", U)), P.lit(-1.0, F64))], to_d)
    out = run(P.projection(src(), [P.col("k"), case], ["k", "c"], [I64, F64]), {"t": t}).sort_by("k")
    assert out.column(1).to_pylist() == [-1.0 if s == "x" else v for s, v in zip(texts, ref_d)]
    # sort key
    out = run(P.sort(src(), [P.sort_expr(to_d)]), {"t": t})
    got_keys = [ref_d[k] for k in out.column("k").to_pylist()]
    non_null = [v for v in got_keys if v is not None]
    assert non_null == sorted(non_null)
    # GROUP BY CAST(d AS STRING) for a double and a decimal(38, 10)
    for col, conv in (("d", lambda i: R.float_to_text(struct.unpack("<Q", struct.pack("<d", dv[i]))[0], 64)),
                      ("m", lambda i: R.decimal_to_text(i % 7, 10))):
        out = run(P.agg(src(), [P.cast(P.col(col), U)], ["g"], [P.agg_expr("COUNT", [P.col("k")], I64)], ["c"], ["PARTIAL"]), {"t": t})
        exp = {}
        for i in range(n):
            exp[conv(i)] = exp.get(conv(i), 0) + 1
        assert dict(zip(out.column(0).to_pylist(), out.column(1).to_pylist())) == exp, col
    # sha256(CAST(d AS STRING))
    out = run(P.projection(src(), [P.col("k"), P.scalar_fn("Spark_Sha256", [P.cast(P.col("d"), U)], U)], ["k", "h"], [I64, U]), {"t": t}).sort_by("k")
    assert out.column(1).to_pylist() == [hashlib.sha256(R.float_to_text(struct.unpack("<Q", struct.pack("<d", v))[0], 64).encode()).hexdigest()
                                         for v in dv]
