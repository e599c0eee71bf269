"""Plain-Python exact references for the operations of the expression VM (k_expr.cu): arithmetic, comparisons, casts, the
decimal functions, the date parts and the date text.

Values use the canonical forms of key_reference.py: integers, dates and timestamps as the stored Python int, floats as their
IEEE bit pattern, decimals as the unscaled int, bool as bool, utf8 as bytes, NULL as None.  Every function takes and returns
canonical values, so a NULL result, a NaN payload and the sign of zero are all compared exactly.  Only Python ints, `struct`
and `math` are used -- no engine, no numpy, no Arrow."""
from __future__ import annotations

import math

from key_reference import DAY_MS, INT_BITS, bits_f32, bits_f64, edge_values, f32_bits, f64_bits, total_order, wrap  # noqa: F401

MAX_PRECISION = 38
MIN_ADJUSTED_SCALE = 6                                   # Spark's DecimalType.MINIMUM_ADJUSTED_SCALE


# -------------------------------------------------------------------------------------------- float helpers
def to_float(v: int, t: str) -> float:
    return bits_f32(v) if t == "float32" else bits_f64(v)


F32_MAX = (2 - 2.0 ** -23) * 2.0 ** 127


def from_float(x: float, t: str) -> int:
    """the bits of x rounded to type t (float32: one rounding of the f64 value, through struct; past the float32 range the
    value rounds to the largest finite value or to infinity, the tie 2^128 - 2^103 going to infinity)"""
    if t == "float64":
        return f64_bits(x)
    if math.isfinite(x) and abs(x) > F32_MAX:
        return f32_bits(math.copysign(math.inf if abs(x) >= 2.0 ** 128 - 2.0 ** 103 else F32_MAX, x))
    return f32_bits(x)


def int_to_float(v: int, t: str) -> int:
    """an exact integer rounded once to type t (half to even), as a direct int64 -> float conversion does"""
    if t == "float64":
        return f64_bits(float(v))                            # Python rounds an int to a double correctly
    a = abs(v)
    if a >= 1 << 24:
        sh = a.bit_length() - 24
        q, r = divmod(a, 1 << sh)
        if 2 * r > 1 << sh or (2 * r == 1 << sh and q & 1):
            q += 1
        a = q << sh
    return from_float(float(a) if v >= 0 else -float(a), t)


def _fdiv(x: float, y: float) -> float:
    """IEEE division, including x / 0 (Python raises there)"""
    if y == 0.0:
        if math.isnan(x) or x == 0.0:
            return math.nan
        return math.copysign(math.inf, x) * math.copysign(1.0, y)
    return x / y


# -------------------------------------------------------------------------------------------- arithmetic
def arith(op: str, a, b, t: str):
    """Plus / Minus / Multiply / Divide / Modulo and the bitwise ops on two values of type t.  Integers wrap at their width
    (MIN / -1 = MIN), `%` takes the sign of the dividend, a zero divisor gives NULL (the divisor goes through NullIfZero), shift
    counts are masked by 31 (int8 / int16 / int32) or 63 (int64).  float32 is computed in f64 and rounded once, exact for + - * /."""
    if a is None or b is None:
        return None
    if t in INT_BITS:
        bits = INT_BITS[t]
        if op == "Plus":
            r = a + b
        elif op == "Minus":
            r = a - b
        elif op == "Multiply":
            r = a * b
        elif op in ("Divide", "Modulo"):
            if b == 0:
                return None
            q = abs(a) // abs(b) * (1 if (a < 0) == (b < 0) else -1)     # truncating division
            r = q if op == "Divide" else a - q * b
            if op == "Modulo" and b == -1:
                r = 0
            elif op == "Divide" and b == -1:
                r = -a                                                 # wraps for MIN
        elif op == "BitwiseAnd":
            r = a & b
        elif op == "BitwiseOr":
            r = a | b
        elif op == "BitwiseXor":
            r = a ^ b
        elif op in ("BitwiseShiftLeft", "BitwiseShiftRight"):
            s = b & (63 if bits == 64 else 31)
            # the shift runs on the int64 register: int8 / int16 shifted left wrap to their own width afterwards
            r = wrap(a << s, 64) if op == "BitwiseShiftLeft" else a >> s
        else:
            raise ValueError(op)
        return wrap(r, bits)
    if t in ("float32", "float64"):
        x, y = to_float(a, t), to_float(b, t)
        if op == "Plus":
            r = x + y
        elif op == "Minus":
            r = x - y
        elif op == "Multiply":
            r = x * y
        elif op == "Divide":
            r = _fdiv(x, y)
        elif op == "Modulo":
            r = math.fmod(x, y) if y != 0 and not math.isinf(x) else (x if math.isinf(y) and not math.isinf(x) else math.nan)
        else:
            raise ValueError(op)
        return from_float(r, t)
    raise ValueError(t)


def negate(a, t: str):
    if a is None:
        return None
    if t in INT_BITS:
        return wrap(-a, INT_BITS[t])
    return a ^ (1 << (31 if t == "float32" else 63))               # flips the sign bit, NaN included


def compare(op: str, a, b, t: str):
    """Eq / NotEq / Lt / LtEq / Gt / GtEq (NULL in, NULL out) and IsNotDistinctFrom; floats in IEEE total order (NaN == NaN,
    -0.0 < +0.0)"""
    if op == "IsNotDistinctFrom":
        if a is None or b is None:
            return a is None and b is None
    elif a is None or b is None:
        return None
    if t in ("float32", "float64"):
        w = 32 if t == "float32" else 64
        a, b = total_order(a, w), total_order(b, w)
    c = (a > b) - (a < b)
    return {"Eq": c == 0, "NotEq": c != 0, "Lt": c < 0, "LtEq": c <= 0, "Gt": c > 0, "GtEq": c >= 0, "IsNotDistinctFrom": c == 0}[op]


def kleene_and(a, b):
    if a is False or b is False:
        return False
    return None if a is None or b is None else True


def kleene_or(a, b):
    if a is True or b is True:
        return True
    return None if a is None or b is None else False


# -------------------------------------------------------------------------------------------- decimals
def round_half_away(num: int, den: int) -> int:
    """num / den rounded half away from zero (den > 0)"""
    q, r = divmod(abs(num), den)
    if 2 * r >= den:
        q += 1
    return q if num >= 0 else -q


def fits(v: int, precision: int) -> bool:
    return abs(v) < 10 ** precision


def rescale(v, s_from: int, p_to: int, s_to: int):
    """decimal -> decimal: exact when the scale grows, half away from zero when it shrinks; NULL when the result has more than
    p_to digits (change_precision_round_half_up, spark_check_overflow.rs)"""
    if v is None:
        return None
    r = v * 10 ** (s_to - s_from) if s_to >= s_from else round_half_away(v, 10 ** (s_from - s_to))
    return r if fits(r, p_to) else None


check_overflow = rescale                                 # Spark_CheckOverflow(x: (p, s_from)) -> (p_to, s_to); Spark: NULL on overflow


def make_decimal(v, precision: int, null_on_overflow: bool = True):
    """Spark_MakeDecimal: the int64 becomes the unscaled value.  Spark gives NULL when it does not fit the precision; the
    reference (spark_make_decimal.rs) passes it through (null_on_overflow=False)."""
    if v is None:
        return None
    return None if null_on_overflow and not fits(v, precision) else v


def unscaled_value(v):
    """Spark_UnscaledValue: the low 64 bits of the unscaled value, signed"""
    return None if v is None else wrap(v, 64)


def adjust_precision_scale(precision: int, scale: int) -> tuple[int, int]:
    """Spark's DecimalType.adjustPrecisionScale (spark.sql.decimalOperations.allowPrecisionLoss = true)"""
    if precision <= MAX_PRECISION:
        return precision, scale
    if scale < 0:
        return MAX_PRECISION, scale
    int_digits = precision - scale
    return MAX_PRECISION, max(MAX_PRECISION - int_digits, min(scale, MIN_ADJUSTED_SCALE))


def result_decimal_type(op: str, p1: int, s1: int, p2: int, s2: int) -> tuple[int, int]:
    """resultDecimalType of the reference's NativeConverters for Add / Subtract / Multiply"""
    if op == "Multiply":
        return adjust_precision_scale(p1 + p2 + 1, s1 + s2)
    s = max(s1, s2)
    return adjust_precision_scale(max(p1 - s1, p2 - s2) + s + 1, s)


def engine_arith_type(op: str, p1: int, s1: int, p2: int, s2: int) -> tuple[int, int]:
    """the type the engine declares for a decimal sum, difference or product (arrow's rule, capped at 38 digits); operands of a
    sum or difference are first brought to one scale"""
    if op == "Multiply":
        return min(38, p1 + p2 + 1), s1 + s2
    s = max(s1, s2)
    if s1 != s2:
        common = min(38, max(p1 - s1, p2 - s2) + s)
        p1 = p1 if s1 == s else common
        p2 = p2 if s2 == s else common
    return min(38, max(p1, p2) + 1), s


def decimal_binary(op: str, a, sa: int, b, sb: int, p_out: int):
    """Plus / Minus / Multiply of unscaled decimals: exact, NULL when the result has more than p_out digits (Spark's non-ANSI
    arithmetic).  Plus / Minus rescale to the larger scale first; a product is at scale sa + sb."""
    if a is None or b is None:
        return None
    if op == "Multiply":
        r = a * b
    else:
        s = max(sa, sb)
        a, b = a * 10 ** (s - sa), b * 10 ** (s - sb)
        r = a + b if op == "Plus" else a - b
    return r if fits(r, p_out) else None


def spark_decimal_op(op: str, a, p1: int, s1: int, b, p2: int, s2: int):
    """the reference's plan Cast(BinaryExpr(Cast(lhs, rt), rhs), rt) evaluated exactly with NULL on overflow; returns the value at
    rt = result_decimal_type(...)"""
    rp, rs = result_decimal_type(op, p1, s1, p2, s2)
    lc = rescale(a, s1, rp, rs)
    if lc is None or b is None:
        return None
    ip, isc = engine_arith_type(op, rp, rs, p2, s2)
    inner = decimal_binary(op, lc, rs, b, s2, ip)
    return rescale(inner, isc, rp, rs)


def round_decimal(v, scale: int, digits: int, half_even: bool = False):
    """Spark_Round / Spark_BRound of an unscaled decimal at `digits` fraction digits; the declared type is kept, so the result is
    rounded at 10^(scale - digits) and stays at `scale`"""
    if v is None:
        return None
    drop = scale - digits
    if drop <= 0:
        return v
    f = 10 ** drop
    q, r = divmod(abs(v), f)
    if 2 * r > f or (2 * r == f and (not half_even or q % 2 == 1)):
        q += 1
    return (q if v >= 0 else -q) * f


def round_int(v, digits: int, half_even: bool = False, bits: int = 64):
    """Spark_Round / Spark_BRound of an integer: unchanged for digits >= 0, else rounded at 10^-digits in i128 and truncated back
    to the type's width (spark_round.rs: `round_i128_half_up(v as i128, scale) as i64`), so round(-2^63, -1) wraps"""
    if v is None or digits >= 0:
        return v
    return wrap(round_decimal(v, 0, digits, half_even), bits)


# -------------------------------------------------------------------------------------------- casts
def cast(v, src: str, dst: str):
    """CAST between the VM's numeric types.  Types: int8..int64, float32 / float64, bool, or ("dec", p, s).
    int -> narrower int and decimal -> int / narrower decimal give NULL out of range (arrow safe cast); float -> int saturates
    and NaN gives 0 (cast.rs); float -> decimal is round_half_away(x * 10.0^s); decimal -> float is float(unscaled) / 10.0^s."""
    if v is None:
        return None
    sd, dd = isinstance(src, tuple), isinstance(dst, tuple)
    if src == "bool":
        v, src = int(v), "int8"
    if dst == "bool":
        if src in ("float32", "float64"):
            return to_float(v, src) != 0.0
        return v != 0
    if src in INT_BITS:
        if dst in INT_BITS:
            b = INT_BITS[dst]
            return v if -(1 << (b - 1)) <= v < (1 << (b - 1)) else None
        if dst in ("float32", "float64"):
            return int_to_float(v, dst)
        if dd:
            r = v * 10 ** dst[2]
            return r if fits(r, dst[1]) else None
    if src in ("float32", "float64"):
        x = to_float(v, src)
        if dst in INT_BITS:
            b = INT_BITS[dst]
            lo, hi = -(1 << (b - 1)), (1 << (b - 1)) - 1
            if math.isnan(x):
                return 0
            if x >= hi:
                return hi
            if x <= lo:
                return lo
            return int(x)                                           # truncation toward zero
        if dst in ("float32", "float64"):
            return from_float(x, dst)
        if dd:
            if math.isnan(x) or math.isinf(x):
                return None
            y = x * 10.0 ** dst[2]                                  # one f64 multiplication, as the kernel does
            if math.isinf(y):
                return None
            f = math.floor(abs(y))
            r = int(f) + (abs(y) - f >= 0.5)                        # half away from zero (Python's round() goes to even)
            r = r if y >= 0 else -r
            return r if fits(r, dst[1]) else None
    if sd:
        s = src[2]
        if dd:
            return rescale(v, s, dst[1], dst[2])
        if dst in INT_BITS:
            q = abs(v) // 10 ** s * (1 if v >= 0 else -1)           # truncation toward zero
            b = INT_BITS[dst]
            return q if -(1 << (b - 1)) <= q < (1 << (b - 1)) else None
        if dst in ("float32", "float64"):
            return from_float(float(v) / 10.0 ** s, dst)
    raise ValueError((src, dst))


# -------------------------------------------------------------------------------------------- NULL handling
def null_if(a, b):
    """NullIf(a, b): NULL where a == b (both non-NULL), else a"""
    return None if a is not None and b is not None and a == b else a


def null_if_zero(a, t: str):
    if a is None:
        return None
    if t in ("float32", "float64"):
        return None if to_float(a, t) == 0.0 else a
    return None if a == 0 else a


def coalesce(*vals):
    return next((v for v in vals if v is not None), None)


def normalize_nan_and_zero(a, t: str):
    """Spark_NormalizeNanAndZero: every NaN becomes the canonical quiet NaN, -0.0 becomes +0.0"""
    if a is None:
        return None
    x = to_float(a, t)
    if math.isnan(x):
        return 0x7FC00000 if t == "float32" else 0x7FF8000000000000
    return 0 if x == 0.0 else a


# -------------------------------------------------------------------------------------------- dates and strings
def civil_from_days(z: int) -> tuple[int, int, int]:
    """proleptic Gregorian (year, month, day) of a day count since 1970-01-01, for any int"""
    z += 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = mp + 3 if mp < 10 else mp - 9
    return yoe + era * 400 + (m <= 2), m, d


def days_from_civil(y: int, m: int, d: int) -> int:
    y -= m <= 2
    era = y // 400
    yoe = y - era * 400
    doy = (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def date_part(days, part: str):
    """year / month / day / quarter / doy / week (ISO-8601) / dayofweek (Spark: Sunday = 1) / dow (date_part: Sunday = 0)"""
    if days is None:
        return None
    y, m, d = civil_from_days(days)
    if part == "year":
        return y
    if part == "month":
        return m
    if part == "day":
        return d
    if part == "quarter":
        return (m - 1) // 3 + 1
    if part == "doy":
        return days - days_from_civil(y, 1, 1) + 1
    if part == "dayofweek":
        return (days + 4) % 7 + 1
    if part == "dow":
        return (days + 4) % 7
    if part == "week":
        thursday = days - (days + 3) % 7 + 3
        return (thursday - days_from_civil(civil_from_days(thursday)[0], 1, 1)) // 7 + 1
    raise ValueError(part)


def date_text(days) -> bytes | None:
    """chrono's NaiveDate text: YYYY-MM-DD for years 0..9999, else the year with its sign and at least four digits ({:+05})"""
    if days is None:
        return None
    y, m, d = civil_from_days(days)
    ys = f"{y:04d}" if 0 <= y <= 9999 else f"{y:+05d}"
    return f"{ys}-{m:02d}-{d:02d}".encode()


def decimal_text(v, scale: int) -> bytes | None:
    """decimal -> utf8 (cast.rs): plain digits with exactly `scale` fraction digits and at least one integer digit"""
    if v is None:
        return None
    s = str(abs(v)).rjust(scale + 1, "0")
    body = s if scale == 0 else s[:-scale] + "." + s[-scale:]
    return ("-" if v < 0 else "").encode() + body.encode()


_ASCII_WS = b" "


def trim(s, which: str = "both"):
    """Trim / Ltrim / Rtrim: removes ASCII spaces only"""
    if s is None:
        return None
    if which in ("both", "left"):
        s = s.lstrip(_ASCII_WS)
    if which in ("both", "right"):
        s = s.rstrip(_ASCII_WS)
    return s


def ascii_upper(s):
    return None if s is None else bytes(c - 32 if 97 <= c <= 122 else c for c in s)


def ascii_lower(s):
    return None if s is None else bytes(c + 32 if 65 <= c <= 90 else c for c in s)


def octet_length(s):
    return None if s is None else len(s)
