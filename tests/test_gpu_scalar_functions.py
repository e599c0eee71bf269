"""greatest, least, nvl2, months_between, date_trunc, make_date, hex, chr, acosh, factorial, RowNum and spark_partition_id on the
GPU, value by value against the plain-Python reference in scalar_reference.py (its docstring states the semantics), at the edges of
every type and in every position the planner accepts them."""
import datetime as dt
import decimal
import hashlib
import math
import struct

import numpy as np
import pyarrow as pa
import pytest

import scalar_reference as R
from auron_b200 import proto as P
from auron_b200 import runtime
from helpers import assert_same_rows, batches, run

pytestmark = pytest.mark.gpu

U, B, I32, I64, F64, D32, BOOL = pa.string(), pa.binary(), pa.int32(), pa.int64(), pa.float64(), pa.date32(), pa.bool_()
TS = pa.timestamp("us")
I64_MIN, I64_MAX, I32_MIN, I32_MAX = -(2**63), 2**63 - 1, -(2**31), 2**31 - 1


def fn(name, *args, t=U):
    return P.scalar_fn(name, list(args), t)


def lit(v, t=U):
    return P.lit(v, t)


def project(t, exprs, types, src=None):
    src = src or P.ffi_reader(t.schema, "t")
    return P.projection(src, exprs, [f"c{i}" for i in range(len(exprs))], types)


def raw(col):
    """values as plain Python: timestamps and dates as integers, utf8 as its bytes, floats as their bit patterns"""
    t = col.type
    if pa.types.is_timestamp(t):
        return col.cast(I64).to_pylist()
    if pa.types.is_date32(t):
        return col.cast(I32).to_pylist()
    if pa.types.is_string(t):
        return col.cast(B).to_pylist()
    if pa.types.is_float64(t):
        return [None if v is None else struct.pack("<d", v) for v in col.to_pylist()]
    if pa.types.is_float32(t):
        return [None if v is None else struct.pack("<f", v) for v in col.to_pylist()]
    return col.to_pylist()


def fbits(v, t):
    if v is None or not (pa.types.is_floating(t)):
        return v
    return struct.pack("<d" if pa.types.is_float64(t) else "<f", v)


def check(got, exp, what):
    assert len(got) == len(exp), what
    bad = [i for i, (a, b) in enumerate(zip(got, exp)) if a != b]
    assert not bad, (what, len(bad), [(i, got[i], exp[i]) for i in bad[:4]])


# ---------------------------------------------------------------------------------------------- greatest / least at the edges
NAN, INF = float("nan"), float("inf")
EDGES = {   # arrow type -> (edge values, order kind of scalar_reference.order_key)
    "int8": (pa.int8(), [-128, 127, 0, -1, 1], "int"),
    "int16": (pa.int16(), [-32768, 32767, 0, -1, 1], "int"),
    "int32": (I32, [I32_MIN, I32_MAX, 0, -1, 1], "int"),
    "int64": (I64, [I64_MIN, I64_MAX, 0, -1, 1, I64_MIN + 1], "int"),
    "float32": (pa.float32(), [NAN, INF, -INF, 0.0, -0.0, 1.5, -1.5, 3.4028234663852886e38, 1e-45], "f32"),
    "float64": (F64, [NAN, INF, -INF, 0.0, -0.0, 1.5, -1.5, 1.7976931348623157e308, 5e-324], "f64"),
    "decimal38": (pa.decimal128(38, 0), [10**38 - 1, -(10**38 - 1), 2**64 + 5, 2 * 2**64 + 5, -(2**64) + 5, -(2 * 2**64) + 5, 5, 0], "int"),
    "date32": (D32, [I32_MIN, I32_MAX, 0, -1, 19000], "int"),
    "ts_s": (pa.timestamp("s"), [I64_MIN, I64_MAX, 0, -1, 1], "int"),
    "ts_ms": (pa.timestamp("ms"), [I64_MIN, I64_MAX, 0, -1, 1], "int"),
    "ts_us": (TS, [I64_MIN, I64_MAX, 0, -1, 1], "int"),
    "ts_ns": (pa.timestamp("ns"), [I64_MIN, I64_MAX, 0, -1, 1], "int"),
    "bool": (BOOL, [True, False], "int"),
    "utf8": (U, ["", "a", "a\x00", "a\x00b", "ab", "ÿ", "ÿa", "\U0010ffff", "\U0010ffffa", "b"], "bytes"),
    "binary": (B, [b"", b"\x00", b"\x00\x00", b"\xff", b"\xff\x00", b"a", b"ab", b"a\xff"], "bytes"),
}


def _edge_column(rng, at, vals, n, p_null):
    """a column of edge values with NULLs, and its values as plain Python (timestamps and dates as integers, utf8 as bytes)"""
    py = [None if m else vals[k] for k, m in zip(rng.integers(0, len(vals), n), rng.random(n) < p_null)]
    if pa.types.is_decimal(at):
        arr = pa.array([None if v is None else decimal.Decimal(v) for v in py], type=at)
    elif pa.types.is_timestamp(at) or pa.types.is_date32(at):
        arr = pa.array(py, type=I64 if pa.types.is_timestamp(at) else I32).cast(at)
    else:
        arr = pa.array(py, type=at)
    return arr, [v.encode() if isinstance(v, str) else v for v in py]


@pytest.mark.parametrize("name", sorted(EDGES))
def test_greatest_and_least_at_the_edges(name):
    at, vals, kind = EDGES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    n = 3000
    cols = [_edge_column(rng, at, vals, n, 0.5 if k < 2 else 0.15) for k in range(12)]   # rows where both of the first two are NULL
    t = pa.table({f"a{k}": c[0] for k, c in enumerate(cols)})
    a = [P.col(f"a{k}") for k in range(12)]
    exprs = [fn("Greatest", a[0], a[1], t=at), fn("Least", a[0], a[1], t=at), fn("Greatest", *a, t=at), fn("Least", *a, t=at),
             fn("Least", a[0], lit(None, at), a[1], t=at)]
    got = run(project(t, exprs, [at] * len(exprs)), {"t": t}, chunk=1100)
    rows = list(zip(*[c[1] for c in cols]))
    refs = [lambda r: R.greatest(r[:2], kind), lambda r: R.greatest(r[:2], kind, least=True), lambda r: R.greatest(r, kind),
            lambda r: R.greatest(r, kind, least=True), lambda r: R.greatest(r[:2], kind, least=True)]
    for k, f in enumerate(refs):
        assert got.schema.field(k).type == at
        check(raw(got.column(k)), [fbits(f(r), at) for r in rows], (name, k))
    assert any(r[0] is None and r[1] is None for r in rows)


# ---------------------------------------------------------------------------------------------- months_between
def utc_us(y, mo, d, h=0, mi=0, s=0):
    return int(dt.datetime(y, mo, d, h, mi, s, tzinfo=dt.timezone.utc).timestamp()) * 1_000_000


ANCHORS = [utc_us(*a) for a in [(2024, 3, 10, 7), (2024, 11, 3, 6), (2018, 11, 4, 3), (2019, 2, 17, 2), (2023, 10, 1, 15),
                                (2024, 4, 7, 15), (2022, 11, 6, 4), (2022, 3, 13, 5), (1986, 1, 1), (1969, 12, 31, 23), (1960, 2, 29, 12),
                                (1905, 6, 30), (2099, 12, 31, 12), (2024, 2, 29), (2024, 1, 31)]]


def _instants(rng, n):
    base = np.array(ANCHORS, dtype=np.int64)[rng.integers(0, len(ANCHORS), n)]
    return base + rng.integers(-4 * 86400 * 10**6, 4 * 86400 * 10**6, n) + rng.integers(0, 1000, n) * (rng.random(n) < 0.3)


@pytest.mark.parametrize("zone", [None, "America/New_York", "Asia/Kathmandu", "Australia/Lord_Howe", "America/Sao_Paulo", "America/Havana"])
def test_months_between_in_zones_and_units(zone):
    rng = np.random.default_rng(7 if zone is None else sum(map(ord, zone)))
    n = 3000
    a_us, b_us = _instants(rng, n), _instants(rng, n)
    if zone == "America/Sao_Paulo":   # 2018-11-04 has no local midnight: the lookup walks forward to 01:00
        a_us[:40] = utc_us(2018, 11, 4, 15) + np.arange(40) * 600 * 10**6
        b_us[:40] = utc_us(2018, 10, 1, 3)
    b_ns = b_us * 1000 + rng.integers(-999, 1000, n)
    c_ms, d_s = a_us // 1000, b_us // 10**6
    e_days = (b_us // (86400 * 10**6)).astype(np.int32)
    nul = lambda: rng.random(n) < 0.05   # noqa: E731
    t = pa.table({"a": pa.array(a_us, mask=nul()).cast(TS), "b": pa.array(b_ns, mask=nul()).cast(pa.timestamp("ns")),
                  "c": pa.array(c_ms, mask=nul()).cast(pa.timestamp("ms")), "d": pa.array(d_s, mask=nul()).cast(pa.timestamp("s")),
                  "e": pa.array(e_days, mask=nul()).cast(D32), "r": pa.array(rng.random(n) < 0.5, mask=nul())})
    z = lit(zone)
    mb = lambda x, y, r: fn("Spark_MonthsBetween", x, y, r, z, t=F64)   # noqa: E731
    a, b, c, d, e, r = P.col("a"), P.col("b"), P.col("c"), P.col("d"), P.col("e"), P.col("r")
    exprs = [mb(a, b, r), mb(c, d, lit(True, BOOL)), mb(e, a, lit(False, BOOL)), mb(a, e, r), mb(b, c, lit(True, BOOL))]
    got = run(project(t, exprs, [F64] * len(exprs)), {"t": t}, chunk=1100)
    col = {k: t.column(k).cast(I64 if k != "e" else I32).to_pylist() if k != "r" else t.column(k).to_pylist() for k in "abcder"}
    ms = {"a": lambda v: R.to_ms(v, "us"), "b": lambda v: R.to_ms(v, "ns"), "c": lambda v: v, "d": lambda v: R.to_ms(v, "s"),
          "e": lambda v: R.to_ms(v, "date32")}

    def ref(x, y, rr):
        return [R.months_between(None if u is None else ms[x](u), None if v is None else ms[y](v), w, zone)
                for u, v, w in zip(col[x], col[y], rr)]
    exps = [ref("a", "b", col["r"]), ref("c", "d", [True] * n), ref("e", "a", [False] * n), ref("a", "e", col["r"]), ref("b", "c", [True] * n)]
    for k, exp in enumerate(exps):
        check(raw(got.column(k)), [fbits(v, F64) for v in exp], (zone, k))
    assert any(v is not None and v < 0 for v in exps[1]) and any(v is not None and v != round(v) for v in exps[0])


# ---------------------------------------------------------------------------------------------- date_trunc
FORMATS = ["YEAR", "yyyy", "YY", "quarter", "MONTH", "mon", "MM", "week", "DAY", "dd", "HOUR", "minute", "SECOND", "MilliSecond",
           "MICROSECOND", "decade", None]


@pytest.mark.parametrize("unit", ["s", "ms", "us", "ns"])
def test_date_trunc_every_level_and_unit(unit):
    rng = np.random.default_rng({"s": 1, "ms": 2, "us": 3, "ns": 4}[unit])
    n = 4000
    per_s = R.UNIT_PER_S[unit]
    v = np.concatenate([np.array([I64_MIN, I64_MAX, 0, -1, 1, I64_MIN + 1, I64_MAX - 1], dtype=np.int64),
                        rng.integers(I64_MIN, I64_MAX, n // 4, dtype=np.int64),                               # far past and future
                        rng.integers(-3 * 10**9, 4 * 10**9, n - n // 4 - 7, dtype=np.int64) * per_s + rng.integers(0, per_s, n - n // 4 - 7)])
    at = pa.timestamp(unit)
    t = pa.table({"v": pa.array(v, mask=rng.random(len(v)) < 0.03).cast(at)})
    exprs = [fn("DateTrunc", lit(f), P.col("v"), t=TS) for f in FORMATS] + [fn("DateTrunc", lit("month"), P.col("v"), t=at)]
    got = run(project(t, exprs, [TS] * len(FORMATS) + [at]), {"t": t}, chunk=1500)
    vals = t.column("v").cast(I64).to_pylist()
    for k, f in enumerate(FORMATS):
        check(raw(got.column(k)), [R.date_trunc(f, x, unit, "us") for x in vals], (unit, f))
    check(raw(got.column(len(FORMATS))), [R.date_trunc("month", x, unit) for x in vals], (unit, "same unit"))
    assert got.schema.field(0).type == TS and got.schema.field(len(FORMATS)).type == at


# ---------------------------------------------------------------------------------------------- make_date, factorial, acosh
def test_make_date_invalid_combinations_and_year_range():
    ys = [-5_877_641, -5_877_642, 5_881_580, 5_881_581, 1970, 2000, 1900, 2024, 2023, 0, -1, I32_MIN, I32_MAX]
    ms = [0, 1, 2, 3, 6, 7, 12, 13, -1, I32_MIN, I32_MAX]
    ds = [0, 1, 11, 12, 22, 23, 28, 29, 30, 31, 32, -1, I32_MAX]
    rows = [(y, m, d) for y in ys for m in ms for d in ds]
    rng = np.random.default_rng(3)
    rows += [(int(y), int(m), int(d)) for y, m, d in zip(rng.integers(-3000, 3000, 5000), rng.integers(0, 14, 5000), rng.integers(0, 33, 5000))]
    rows += [(None, 1, 1), (2000, None, 1), (2000, 1, None)]
    t = pa.table({k: pa.array([r[i] for r in rows], type=I32) for i, k in enumerate("ymd")})
    got = run(project(t, [fn("MakeDate", P.col("y"), P.col("m"), P.col("d"), t=D32)], [D32]), {"t": t}, chunk=2000)
    exp = [R.make_date(*r) for r in rows]
    check(raw(got.column(0)), exp, "make_date")
    assert exp.count(None) > 100 and R.make_date(5_881_580, 7, 11) in exp


def test_factorial_and_acosh():
    ns = [-1, 0, 1, 2, 12, 13, 20, 21, I32_MIN, I32_MAX, None]
    xs = [1.0, 1.0000000000000002, 1.5, 2.0, 10.0, 1e10, 1e300, INF, NAN, 0.5, -1.0, 0.9999999999999999, -INF, 0.0]
    xs += list(np.exp(np.random.default_rng(4).uniform(0, 30, 5000)))
    t = pa.table({"n": pa.array((ns * (len(xs) // len(ns) + 1))[:len(xs)], type=I32), "x": pa.array(xs, type=F64)})
    got = run(project(t, [fn("Factorial", P.col("n"), t=I64), fn("Acosh", P.col("x"), t=F64)], [I64, F64]), {"t": t})
    check(got.column(0).to_pylist(), [R.factorial(v) for v in t.column("n").to_pylist()], "factorial")
    # acosh within 5 ulp of glibc's: the CUDA C Programming Guide gives 3 ulp for acosh, glibc's libm-test-ulps at most 2
    g = got.column(1).to_pylist()
    for x, y in zip(xs, g):
        e = math.acosh(x) if x >= 1 else NAN
        if math.isnan(e) or math.isinf(e):
            assert (math.isnan(y) and math.isnan(e)) or y == e, (x, y, e)
        else:
            bx, by = struct.unpack("<q", struct.pack("<d", e))[0], struct.unpack("<q", struct.pack("<d", y))[0]
            assert abs(bx - by) <= 5, (x, y, e)


# ---------------------------------------------------------------------------------------------- hex and chr
def test_hex_and_chr_at_the_edges_in_every_position():
    ints = [0, -1, 1, 15, 16, 255, 256, I64_MIN, I64_MAX, 65, 127, 128, 129, 191, 192, 255, 256 + 65, -65, -256, 2**32, None]
    strs = ["", "a", "é", "天", "😁", "\U0010ffff", "a\x00b", None, "ÿ", "abc"]
    bins = [b"", b"\x00", b"\xff", b"\x00\xff\x80", b"A", None, b"\xff" * 5]
    n = 3000
    rng = np.random.default_rng(5)
    iv = [ints[k] for k in rng.integers(0, len(ints), n)]
    iv[:len(ints)] = ints
    t = pa.table({"i": pa.array(iv, type=I64), "n": pa.array([None if v is None else (v & 0xFFFFFFFF) - (2**32 if v & 0x80000000 else 0) for v in iv], type=I32),
                  "s": pa.array([strs[k] for k in rng.integers(0, len(strs), n)], type=U), "b": pa.array([bins[k] for k in rng.integers(0, len(bins), n)], type=B)})
    i, nn, s, b = P.col("i"), P.col("n"), P.col("s"), P.col("b")
    exprs = [fn("Hex", i), fn("Hex", nn), fn("Hex", s), fn("Hex", b), fn("Chr", i), fn("Chr", nn),
             fn("Spark_StringConcat", lit("<"), fn("Hex", i), fn("Chr", i), fn("Hex", fn("Upper", s)), lit(">")),
             fn("Spark_StringConcatWs", lit("|"), fn("Chr", i), fn("Hex", b), s),
             fn("Spark_MD5", fn("Hex", s)), fn("Spark_MD5", fn("Chr", i)), fn("Spark_Sha256", fn("Hex", i))]
    got = run(project(t, exprs, [U] * len(exprs)), {"t": t}, chunk=1100)
    I_, N_ = t.column("i").to_pylist(), t.column("n").to_pylist()
    S_, B_ = raw(t.column("s")), t.column("b").to_pylist()
    md5 = lambda v: None if v is None else hashlib.md5(v).hexdigest().encode()   # noqa: E731
    cat = lambda *v: None if any(x is None for x in v) else b"".join(v)   # noqa: E731
    exps = [[R.hex_int(v) for v in I_], [R.hex_int(v) for v in N_], [R.hex_bytes(v) for v in S_], [R.hex_bytes(v) for v in B_],
            [R.chr_(v) for v in I_], [R.chr_(v) for v in N_],
            [cat(b"<", R.hex_int(x), R.chr_(x), R.hex_bytes(upper(y)), b">") for x, y in zip(I_, S_)],
            [b"|".join(v for v in (R.chr_(x), R.hex_bytes(y), z) if v is not None) for x, y, z in zip(I_, B_, S_)],
            [md5(R.hex_bytes(v)) for v in S_], [md5(R.chr_(v)) for v in I_],
            [None if v is None else hashlib.sha256(R.hex_int(v)).hexdigest().encode() for v in I_]]
    for k, exp in enumerate(exps):
        check(raw(got.column(k)), exp, k)


# ---------------------------------------------------------------------------------------------- fuzz
def _fuzz_table(n, seed):
    rng = np.random.default_rng(seed)
    nul = lambda: rng.random(n) < 0.06   # noqa: E731
    words = ["", "a", "ab", "é", "天地", "\U0010ffff", "zz", "a\x00"]
    pick = lambda: [words[k] for k in rng.integers(0, len(words), n)]   # noqa: E731
    t0 = utc_us(1950, 1, 1)
    return pa.table({"i": pa.array(rng.integers(-5, 5, n) * (rng.integers(0, 2, n) * (2**62) + 1), mask=nul()),
                     "j": pa.array(rng.integers(-5, 5, n), mask=nul()), "s": pa.array(pick(), type=U, mask=nul()),
                     "t": pa.array(pick(), type=U, mask=nul()),
                     "y": pa.array(rng.integers(1890, 2110, n).astype(np.int32), mask=nul()), "m": pa.array(rng.integers(0, 14, n).astype(np.int32), mask=nul()),
                     "d": pa.array(rng.integers(0, 33, n).astype(np.int32), mask=nul()), "n": pa.array(rng.integers(-2, 300, n).astype(np.int32), mask=nul()),
                     "ts": pa.array(rng.integers(t0, -t0 + 2 * 10**15, n), mask=nul()).cast(TS),
                     "ts2": pa.array(rng.integers(t0, -t0 + 2 * 10**15, n), mask=nul()).cast(TS),
                     "r": pa.array(rng.random(n) < 0.5, mask=nul()), "k": pa.array(rng.integers(0, 100, n).astype(np.int32))})


def upper(v):   # the VM's ASCII upper / lower
    return None if v is None else bytes(x - 32 if 97 <= x <= 122 else x for x in v)


def lower(v):
    return None if v is None else bytes(x + 32 if 65 <= x <= 90 else x for x in v)


def _fuzz_cases():
    c = P.col
    return [
        # views compare through their upper / lower marks
        (fn("Greatest", fn("Upper", c("s")), fn("Lower", c("t")), t=U), U, lambda r: R.greatest([upper(r["s"]), lower(r["t"])], "bytes")),
        (fn("Greatest", c("i"), c("j"), lit(0, I64), t=I64), I64, lambda r: R.greatest([r["i"], r["j"], 0], "int")),
        (fn("Least", c("s"), c("t"), t=U), U, lambda r: R.greatest([r["s"], r["t"]], "bytes", least=True)),
        (fn("Nvl2", c("i"), c("s"), c("t"), t=U), U, lambda r: R.nvl2(r["i"], r["s"], r["t"])),
        (fn("Nvl2", c("s"), c("i"), c("j"), t=I64), I64, lambda r: R.nvl2(r["s"], r["i"], r["j"])),
        (fn("MakeDate", c("y"), c("m"), c("d"), t=D32), D32, lambda r: R.make_date(r["y"], r["m"], r["d"])),
        (fn("Factorial", c("n"), t=I64), I64, lambda r: R.factorial(r["n"])),
        (fn("DateTrunc", lit("WEEK"), c("ts"), t=TS), TS, lambda r: R.date_trunc("WEEK", r["ts"], "us")),
        (fn("Spark_MonthsBetween", c("ts"), c("ts2"), c("r"), lit("Australia/Lord_Howe"), t=F64), F64,
         lambda r: fbits(R.months_between(None if r["ts"] is None else R.to_ms(r["ts"], "us"), None if r["ts2"] is None else R.to_ms(r["ts2"], "us"),
                                          r["r"], "Australia/Lord_Howe"), F64)),
        (fn("Hex", c("i")), U, lambda r: R.hex_int(r["i"])),
        (fn("Spark_StringConcat", fn("Chr", c("n")), fn("Hex", c("s"))), U,
         lambda r: None if r["n"] is None or r["s"] is None else R.chr_(r["n"]) + R.hex_bytes(r["s"])),
    ]


def _rows(t):
    cols = {k: raw(t.column(k)) for k in t.column_names}
    return [dict(zip(cols, v)) for v in zip(*cols.values())]


def _check_fuzz(got, t, cases):
    rows = _rows(t)
    assert got.num_rows == len(rows)
    for k, (_, typ, ref) in enumerate(cases):
        assert got.schema.field(k).type == typ, k
        check(raw(got.column(k)), [ref(r) for r in rows], k)


def test_fuzz_several_batches():
    t = _fuzz_table(200_000, seed=61)
    cases = _fuzz_cases()
    got = run(project(t, [c[0] for c in cases], [c[1] for c in cases]), {"t": t}, chunk=70_000)
    _check_fuzz(got, t, cases)


def test_fuzz_below_a_filter():
    t = _fuzz_table(60_000, seed=62)
    cases = _fuzz_cases()
    flt = P.filter_(P.ffi_reader(t.schema, "t"), [P.binary("Lt", P.col("k"), lit(37, I32))])
    got = run(project(t, [c[0] for c in cases], [c[1] for c in cases], src=flt), {"t": t}, chunk=25_000)
    _check_fuzz(got, t.filter(pa.array(np.asarray(t.column("k")) < 37)), cases)


# ---------------------------------------------------------------------------------------------- other positions
def test_greatest_and_nvl2_in_a_filter_and_case():
    t = _fuzz_table(50_000, seed=63)
    rows = _rows(t)
    i, j, s, tt = P.col("i"), P.col("j"), P.col("s"), P.col("t")
    src = P.ffi_reader(t.schema, "t")
    g = fn("Greatest", i, j, t=I64)
    preds = [([P.binary("Gt", g, lit(0, I64))], lambda r: (R.greatest([r["i"], r["j"]], "int") or 0) > 0),
             ([P.binary("Lt", fn("Nvl2", s, i, j, t=I64), lit(2, I64))], lambda r: (v := R.nvl2(r["s"], r["i"], r["j"])) is not None and v < 2),
             ([P.binary("Eq", fn("Least", s, tt, t=U), lit("a"))], lambda r: R.greatest([r["s"], r["t"]], "bytes", least=True) == b"a"),
             ([P.binary("Eq", fn("Upper", s), lit("AB"))], lambda r: upper(r["s"]) == b"AB")]
    for k, (pred, ref) in enumerate(preds):
        got = run(project(t, [i], [I64], src=P.filter_(src, pred)), {"t": t}, chunk=20_000)
        exp = [r["i"] for r in rows if ref(r)]
        assert got.column(0).to_pylist() == exp, k
        assert 0 < len(exp) < len(rows), k
    case = P.case([(P.binary("Gt", g, lit(0, I64)), fn("Nvl2", i, s, tt))], fn("Least", s, tt))
    got = run(project(t, [case], [U]), {"t": t}, chunk=20_000)
    exp = [R.nvl2(r["i"], r["s"], r["t"]) if (R.greatest([r["i"], r["j"]], "int") or 0) > 0 else R.greatest([r["s"], r["t"]], "bytes", least=True)
           for r in rows]
    check(raw(got.column(0)), exp, "case")


def test_greatest_and_nvl2_as_group_by_keys_partial_and_final():
    t = _fuzz_table(120_000, seed=64)
    rows = _rows(t)
    src = P.ffi_reader(t.schema, "t")
    keys = [fn("Greatest", P.col("j"), lit(-2, I64), t=I64), fn("Nvl2", P.col("i"), P.col("s"), lit("none"))]
    partial = P.agg(src, keys, ["g", "v"], [P.agg_expr("COUNT", [P.col("k")], I64)], ["c"], ["PARTIAL"])
    final = P.agg(partial, [P.col("g"), P.col("v")], ["g", "v"], [P.agg_expr("COUNT", [P.lit(None, pa.null())], I64)], ["c"], ["FINAL"])
    got = run(final, {"t": t}, chunk=40_000)
    counts = {}
    for r in rows:
        k = (R.greatest([r["j"], -2], "int"), R.nvl2(r["i"], r["s"], b"none"))
        counts[k] = counts.get(k, 0) + 1
    exp = pa.table({"g": pa.array([k[0] for k in counts], type=I64), "v": pa.array([None if k[1] is None else k[1].decode() for k in counts], type=U),
                    "c": pa.array(list(counts.values()), type=I64)})
    assert_same_rows(got, exp)


# ---------------------------------------------------------------------------------------------- RowNum and spark_partition_id
def test_row_num_across_batches_filters_and_tasks():
    n = 100_000
    rng = np.random.default_rng(65)
    t = pa.table({"i": pa.array(np.arange(n)), "k": pa.array(rng.integers(0, 100, n).astype(np.int32))})
    exprs = [P.row_num(), P.col("i"), P.binary("Plus", P.row_num(), lit(1000, I64))]
    plan = project(t, exprs, [I64] * 3)
    for _ in range(2):   # every task counts from 0
        got = run(plan, {"t": t}, chunk=30_000)
        assert got.column(0).to_pylist() == list(range(n))
        assert got.column(2).to_pylist() == [v + 1000 for v in range(n)]
    flt = P.filter_(P.ffi_reader(t.schema, "t"), [P.binary("Lt", P.col("k"), lit(37, I32))])
    got = run(project(t, exprs, [I64] * 3, src=flt), {"t": t}, chunk=30_000)
    kept = np.flatnonzero(np.asarray(t.column("k")) < 37)
    assert got.column(1).to_pylist() == kept.tolist()
    assert got.column(0).to_pylist() == list(range(len(kept)))
    assert got.column(2).to_pylist() == [v + 1000 for v in range(len(kept))]


def test_spark_partition_id_of_two_partitions():
    t = pa.table({"i": pa.array(np.arange(5000))})
    src = P.ffi_reader(t.schema, "t")
    for pid in (0, 5):
        plan = project(t, [P.spark_partition_id(), P.col("i")], [I32, I64],
                       src=P.filter_(src, [P.binary("Eq", P.spark_partition_id(), lit(pid, I32))]))
        got = runtime.run_task(P.task_definition(plan, stage_id=1, partition_id=pid, task_id=pid), {"t": batches(t, 2000)})
        assert got.column(0).to_pylist() == [pid] * 5000 and got.column(0).null_count == 0
        assert got.schema.field(0).type == I32
