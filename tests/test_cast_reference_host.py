"""CPU checks of CAST between utf8 and float / double / boolean and of CAST(float / double / decimal(38, s) AS STRING): the plain-
Python reference (cast_reference.py) against Java and reference goldens and against Python's float() / repr where the two
specifications agree; the parse and format code the device runs, executed on the host through auron_b200_text_to_float /
auron_b200_float_to_text, against the reference; and the planner, through runtime.explain, accepting every position."""
import ctypes as C
import math
import random
import struct

import numpy as np
import pyarrow as pa
import pytest

import cast_reference as R
from auron_b200 import proto as P
from auron_b200 import runtime

U = pa.string()


def d2b(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def b2d(b):
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def f2b(x):   # exact for values that are float32 already
    return struct.unpack("<I", struct.pack("<f", x))[0]


def _lib():
    L = runtime.lib()
    L.auron_b200_float_to_text.restype = C.c_int
    L.auron_b200_float_to_text.argtypes = [C.c_int32, C.c_uint64, C.c_char_p]
    L.auron_b200_text_to_float.restype = C.c_int
    L.auron_b200_text_to_float.argtypes = [C.c_int32, C.c_char_p, C.c_int64, C.POINTER(C.c_uint64)]
    return L


_BUF = C.create_string_buffer(64)


def native_format(x, bits):
    n = _lib().auron_b200_float_to_text(bits, x, _BUF)
    assert n > 0
    return _BUF.raw[:n].decode()


def native_parse(text, bits):
    b = text.encode("utf-8") if isinstance(text, str) else text
    out = C.c_uint64()
    r = _lib().auron_b200_text_to_float(bits, b, len(b), C.byref(out))
    assert r in (0, 1)
    return out.value if r else None


# ------------------------------------------------------------------------------------------------------------ reference
JAVA_DOUBLE = [   # Double.toString, JDK 19+ (a list: 0.0 and -0.0 are one dict key)
    (0.1 + 0.2, "0.30000000000000004"), (1e23, "1.0E23"), (5e-324, "4.9E-324"), (1e-323, "9.9E-324"),
    (2.2250738585072014e-308, "2.2250738585072014E-308"), (9999999.0, "9999999.0"), (1.23456789e7, "1.23456789E7"), (100.0, "100.0"),
    (0.001, "0.001"), (1234567.0, "1234567.0"), (1e7, "1.0E7"), (1e-4, "1.0E-4"), (1.7976931348623157e308, "1.7976931348623157E308"),
    (-1.5, "-1.5"), (0.0, "0.0"), (-0.0, "-0.0"), (math.inf, "Infinity"), (-math.inf, "-Infinity"), (math.nan, "NaN"),
]
JAVA_FLOAT = {3.4028234663852886e38: "3.4028235E38", 16777216.0: "1.6777216E7", 1.401298464324817e-45: "1.4E-45", 0.1: "0.1"}
SPECIALS = {"+NaN": math.nan, "nan": math.nan, "NAN": math.nan, "INF": math.inf, "+nan": None, "-Infinity": -math.inf,
            "Infinity": math.inf, "-inf": -math.inf, "+infinity": math.inf, "1.5d": 1.5, "1.5F": 1.5, "1e400": math.inf,
            "-1e-400": -0.0, "\t 2.5 \n": 2.5, ".5": 0.5, "5.": 5.0, "": None, ".": None, "e5": None, "1e": None, "1.5 d": None,
            "1_0": None, "0x1.8p1": None, " 1": None, "١": None, "1e+": None, "--1": None, "Infinityd": None}


def test_java_goldens():
    for x, s in JAVA_DOUBLE:
        assert R.float_to_text(d2b(x), 64) == s, x
        assert native_format(d2b(x), 64) == s, x
    for x, s in JAVA_FLOAT.items():
        assert R.float_to_text(f2b(x), 32) == s, x
        assert native_format(f2b(x), 32) == s, x
    for text, v in SPECIALS.items():
        for bits in (64, 32):
            got = R.to_float(text, bits)
            assert native_parse(text, bits) == got, (text, bits)
            if v is None:
                assert got is None, text
            elif math.isnan(v):
                assert got == R.NAN[bits], text
            else:
                assert got == (d2b(v) if bits == 64 else f2b(v)), text


def test_reference_goldens():
    # cast.rs test_ok_2 / test_ok_3 (datafusion-ext-exprs): utf8 -> float32
    for text, v in [("123", 123.0), ("321.9", 321.9), ("-098", -98.0), ("sda", None), ("123.4", 123.4)]:
        exp = None if v is None else f2b(v)   # (these values round the same through a double)
        assert R.to_float(text, 32) == exp and native_parse(text, 32) == exp, text
    # cast.rs:660-690 (datafusion-ext-commons): decimal(38, 18) -> utf8
    e18 = 10**18
    assert [R.decimal_to_text(v, 18) for v in [None, 123 * e18, 987 * e18, 987654321 * 10**12, (2**31 - 1) * e18, -(2**31) * e18]] == [
        None, "123.000000000000000000", "987.000000000000000000", "987.654321000000000000", "2147483647.000000000000000000",
        "-2147483648.000000000000000000"]
    assert R.decimal_to_text(-(10**38 - 1), 38) == "-0." + "9" * 38 and R.decimal_to_text(5, 0) == "5" and R.decimal_to_text(-5, 3) == "-0.005"


def test_bool_parsing():
    for t in ["t", "TRUE", " yes\t", "Y", "1", "\x7ftrue\x01"]:
        assert R.to_bool(t) is True, t
    for t in ["f", "False", "n", "NO", "0", " 0 "]:
        assert R.to_bool(t) is False, t
    for t in ["", "2", "tr", "yess", " true", "on", None]:
        assert R.to_bool(t) is None, t


def test_reference_agrees_with_python_where_the_specifications_agree():
    rng = random.Random(5)
    for _ in range(3000):
        x = b2d(rng.getrandbits(64))
        if math.isnan(x) or math.isinf(x):
            continue
        s = R.float_to_text(d2b(x), 64)
        assert float(s) == x, s   # round trip
        mant = repr(abs(x)).split("e")[0].replace(".", "").strip("0")
        if len(mant) >= 2:   # a one-digit shortest may differ: Java considers two digits there
            assert s.lstrip("-").split("E")[0].replace(".", "").strip("0") == mant, (x, s)
        t = "%.*e" % (rng.randint(0, 25), x)
        assert R.to_float(t, 64) == d2b(float(t)), t


# ------------------------------------------------------------------------------------------------ the device code on the host
def _patterns(rng, bits, n):
    mb = 52 if bits == 64 else 23
    special = [0, 1, 2, 3, (1 << mb) - 1, 1 << mb, (1 << mb) + 1]
    special += [(e << mb) for e in range(1, (1 << (bits - 1 - mb)) - 1)]                       # powers of two
    if bits == 64:
        special += [d2b(10.0**k) for k in range(-323, 309)] + [d2b(2.0**53 - 1), d2b(2.0**53), d2b(2.0**53 + 2)]
    else:
        special += [f2b(v) for v in (1e-45, 1e-38, 1e38, 16777215.0, 16777216.0)]
    out = [b | (rng.getrandbits(1) << (bits - 1)) for b in special]
    while len(out) < n:
        b = rng.getrandbits(bits)
        if rng.random() < 0.2:   # subnormals
            b &= (1 << (bits - 1)) | ((1 << mb) - 1)
        out.append(b)
    return out


def _java_layout(neg, digits, x):
    """Java's layout of the decimal 0.d1d2... * 10^(x + 1): `digits` without trailing zeros, x the exponent of the first digit"""
    if -3 <= x < 7:
        out = (digits[:x + 1].ljust(x + 1, "0") + "." + (digits[x + 1:] or "0")) if x >= 0 else "0." + "0" * (-x - 1) + digits
    else:
        out = f"{digits[0]}.{digits[1:] or '0'}E{x}"
    return ("-" if neg else "") + out


def _from_shortest(neg, sci):
    """Java's text from a shortest round-tripping decimal in scientific notation ("d.ddde±x")"""
    mant, _, ex = sci.partition("e")
    digits = mant.replace(".", "").rstrip("0")
    return _java_layout(neg, digits, int(ex)), len(digits)


@pytest.mark.parametrize("bits", [64, 32])
def test_native_format_over_a_million_patterns(bits):
    """Every pattern against an independent shortest-digit generator -- numpy's Dragon4 in unique mode, the closest of the shortest
    decimals -- laid out the Java way; where the shortest has one digit Java also considers two,
    so those go to the reference, as do every power of two (the irregular spacing below them) and every 50th pattern."""
    rng = random.Random(bits)
    mb = 52 if bits == 64 else 23
    emask = (1 << (bits - 1 - mb)) - 1
    to_ref = {b | s for b in [e << mb for e in range(1, emask)] for s in (0, 1 << (bits - 1))}   # every power of two, both signs
    for k, b in enumerate(list(to_ref) + _patterns(rng, bits, 1_000_000)):
        s = native_format(b, bits)
        ab = b & ((1 << (bits - 1)) - 1)
        if ab >> mb == emask or ab == 0:
            assert s == R.float_to_text(b, bits), hex(b)
            continue
        neg = bool(b >> (bits - 1))
        x = np.uint64(ab).view(np.float64) if bits == 64 else np.uint32(ab).view(np.float32)
        sci = np.format_float_scientific(x, unique=True, trim="-")
        exp, n = _from_shortest(neg, sci.replace("e+", "e"))
        if n >= 2 and b not in to_ref and k % 50:
            assert s == exp, (hex(b), s, exp)
        else:
            assert s == R.float_to_text(b, bits), hex(b)
        assert native_parse(s, bits) == b, (hex(b), s)   # parse(format(x)) == x


def _hard_strings(rng):
    out = ["2.2250738585072011e-308", "2.2250738585072012e-308", "2.4703282292062327e-324", "2.4703282292062328e-324",
           "1.7976931348623158e308", "1.7976931348623159e308", "9007199254740993", "9007199254740993.0000000000000000000001",
           "7.038531e-26", "1.00000005960464477539062499", "1.000000059604644775390625", "3.4028235677973366e38",
           "1.4012984643248170709e-45", "7.0064923216240853546e-46", "7.0064923216240853547e-46"]
    # 800-digit halfway strings between neighbouring doubles and floats, with and without a final nonzero digit
    for bits in (64, 32):
        for _ in range(40):
            b = rng.getrandbits(bits - 2) + 1
            _, lo = R.bits_value(b, bits)
            _, hi = R.bits_value(b + 1, bits)
            h = (lo + hi) / 2
            txt = f"{h.numerator * 10**850 // h.denominator}e-850"
            out += [txt, txt + "1", txt.replace("e-850", "0000001e-857")]
    return out


def test_native_parse_against_the_reference():
    rng = random.Random(11)
    texts = _hard_strings(rng)
    while len(texts) < 200_000:
        r = rng.random()
        if r < 0.3:
            texts.append("%.*e" % (rng.randint(0, 19), b2d(rng.getrandbits(63))))
        elif r < 0.5:
            texts.append(repr(b2d(rng.getrandbits(63))))
        elif r < 0.6:
            texts.append("".join(rng.choice("0123456789") for _ in range(rng.randint(20, 60))) + "e" + str(rng.randint(-360, 330)))
        elif r < 0.7:
            texts.append(rng.choice(list(SPECIALS)) + rng.choice(["", " ", "0"]))
        else:
            texts.append("%.*g" % (rng.randint(1, 12), rng.uniform(-1e10, 1e10)))
    for t in texts:
        for bits in (64, 32):
            assert native_parse(t, bits) == R.to_float(t, bits), (t, bits)


def test_bad_arguments():
    L = _lib()
    out = C.c_uint64()
    assert L.auron_b200_text_to_float(16, b"1", 1, C.byref(out)) == -1
    assert L.auron_b200_text_to_float(64, b"1", -1, C.byref(out)) == -1
    assert L.auron_b200_float_to_text(32, 1 << 40, _BUF) == -1
    assert L.auron_b200_float_to_text(8, 0, _BUF) == -1


# ------------------------------------------------------------------------------------------------------------ planning
SCHEMA = pa.schema([("s", U), ("f", pa.float64()), ("g", pa.float32()), ("d", pa.decimal128(38, 10)), ("k", pa.int64()), ("b", pa.binary())])


def _explain(plan):
    return runtime.explain(P.task_definition(plan))


def _src():
    return P.ffi_reader(SCHEMA, "t")


def test_positions_are_accepted():
    F64, BOOL = pa.float64(), pa.bool_()
    to_d = P.try_cast(P.col("s"), F64)
    trimmed = P.cast(P.scalar_fn("Trim", [P.col("s")], U), pa.float32())
    plans = [
        P.projection(_src(), [to_d, trimmed, P.cast(P.col("s"), BOOL), P.try_cast(P.lit("123.4", U), pa.float32())], ["a", "b", "c", "e"],
                     [F64, pa.float32(), BOOL, pa.float32()]),
        P.filter_(_src(), [P.binary("Gt", to_d, P.lit(1.5, F64))]),
        P.projection(_src(), [P.cast(P.col("f"), U), P.cast(P.col("g"), U), P.cast(P.col("d"), U)], ["x", "y", "z"], [U, U, U]),
        P.agg(_src(), [P.cast(P.col("s"), BOOL)], ["k"], [P.agg_expr("SUM", [to_d], F64)], ["s"], ["PARTIAL"]),
        P.agg(_src(), [P.cast(P.col("f"), U)], ["k"], [P.agg_expr("COUNT", [P.col("k")], pa.int64())], ["c"], ["PARTIAL"]),
        P.agg(_src(), [P.cast(P.col("d"), U)], ["k"], [P.agg_expr("COUNT", [P.col("k")], pa.int64())], ["c"], ["PARTIAL"]),
        P.sort(_src(), [P.sort_expr(to_d)]),
        P.projection(_src(), [P.scalar_fn("Spark_Sha256", [P.cast(P.col("f"), U)], U)], ["h"], [U]),
        P.projection(_src(), [P.scalar_fn("Spark_StringConcat", [P.col("s"), P.cast(P.col("d"), U)], U)], ["h"], [U]),
    ]
    for plan in plans:
        assert _explain(plan)


def test_rejections_name_the_cast():
    with pytest.raises(runtime.AuronError, match="binary -> float64"):
        _explain(P.projection(_src(), [P.cast(P.col("b"), pa.float64())], ["a"], [pa.float64()]))
    # only an explicit CAST / TRY_CAST parses text: a coercion the compiler would insert (a math function's argument, a CASE branch) does not
    with pytest.raises(runtime.AuronError, match="utf8 -> float64"):
        _explain(P.projection(_src(), [P.scalar_fn("Sqrt", [P.col("s")], pa.float64())], ["a"], [pa.float64()]))
    with pytest.raises(runtime.AuronError, match="utf8 -> float64"):
        _explain(P.projection(_src(), [P.case([(P.binary("Gt", P.col("k"), P.lit(0, pa.int64())), P.col("f"))], P.col("s"))], ["a"], [pa.float64()]))
    with pytest.raises(runtime.AuronError, match="Spark_StringConcat"):   # float pieces are not built yet
        _explain(P.projection(_src(), [P.scalar_fn("Spark_StringConcat", [P.col("s"), P.cast(P.col("f"), U)], U)], ["h"], [U]))
