"""Spark's non-ANSI CAST between utf8 and float / double / boolean, and of decimal(p <= 38, s >= 0) to utf8, restated in plain
Python with exact arithmetic (fractions.Fraction and integers; no numpy or Arrow).  None stands for NULL.  Floats are bit
patterns (int) of width `bits` (32 or 64).

  * to_float(text, bits): Cast.castToDouble / castToFloat: Java's Double.parseDouble / Float.parseFloat after String.trim
    (characters <= U+0020 at both ends): [+-] then NaN | Infinity (exact case) | digits[.digits] or .digits with an optional
    (e|E)[+-]digits and an optional f F d D suffix.  Otherwise the trimmed text lower-cased: inf, +inf, infinity, +infinity
    -> +inf; -inf, -infinity -> -inf; nan -> NaN.  Anything else is NULL, hexadecimal significands included (Java accepts
    them).  The result is the decimal's value correctly rounded once to the target width (nearest, ties to even).
  * to_bool(text): StringUtils.isTrueString / isFalseString after trimming ASCII whitespace and control characters (<= U+0020
    and U+007F): t true y yes 1 / f false n no 0, ASCII case ignored, else NULL.
  * float_to_text(x, bits): Double.toString / Float.toString as specified since JDK 19: among the decimals that round to x
    the shortest (length 1 or 2 when the shortest has one digit), the one closest to x, ties to an even significand; plain
    notation for 10^-3 <= |d| < 10^7, else d.ddd...E[-]n.
  * decimal_to_text(unscaled, scale): plain digits, at least "0" before the point, exactly `scale` fractional digits, '-'.
"""
import re
from fractions import Fraction

FORMATS = {64: (52, 1023), 32: (23, 127)}   # explicit significand bits, exponent bias
NAN = {64: 0x7FF8000000000000, 32: 0x7FC00000}
_DEC = re.compile(r"([+-]?)(\d+(?:\.\d*)?|\.\d+)(?:[eE]([+-]?\d+))?[fFdD]?\Z")


def inf_bits(bits):
    mb, _ = FORMATS[bits]
    return ((1 << (bits - 1 - mb)) - 1) << mb


def round_to_bits(v, bits):
    """the bit pattern of the non-negative rational v rounded to nearest, ties to even"""
    mb, bias = FORMATS[bits]
    if v == 0:
        return 0
    e = v.numerator.bit_length() - v.denominator.bit_length()
    if Fraction(2) ** e > v:
        e -= 1
    e = max(e, 1 - bias)                      # subnormals share the least exponent
    scaled = v / Fraction(2) ** (e - mb)      # significand at 2^(e - mb)
    m = scaled.numerator // scaled.denominator
    rem = scaled - m
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and m & 1):
        m += 1
    # the implicit bit carries into the exponent field, so does a significand rounded up to 2^(mb + 1)
    b = ((e + bias - 1) << mb) + m if m >> mb else m
    return min(b, inf_bits(bits))


def to_float(text, bits):
    if text is None:
        return None
    if isinstance(text, bytes):
        text = text.decode("latin-1")
    t = text.strip("".join(chr(c) for c in range(0x21)))
    sign_bit = 1 << (bits - 1)
    body = t[1:] if t[:1] in "+-" else t
    neg = t[:1] == "-"
    if body == "NaN":
        return NAN[bits]
    if body == "Infinity":
        return (sign_bit if neg else 0) | inf_bits(bits)
    m = _DEC.match(t)
    if not m or not all(c.isascii() for c in t):
        low = "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in t)
        if low in ("inf", "+inf", "infinity", "+infinity"):
            return inf_bits(bits)
        if low in ("-inf", "-infinity"):
            return sign_bit | inf_bits(bits)
        if low == "nan":
            return NAN[bits]
        return None
    digits = m.group(2)
    ip, _, fp = digits.partition(".")
    es = (m.group(3) or "0").lstrip("+")
    eneg = es.startswith("-")
    es = es.lstrip("-").lstrip("0") or "0"
    ex = (-1 if eneg else 1) * (10**12 if len(es) > 12 else int(es))   # beyond any text's number of digits: saturate
    ds = (ip + fp).lstrip("0")
    e10 = ex - len(fp)   # value = int(ds) * 10^e10
    if len(ds) > 800:   # halfway points have at most 767 significant digits: the rest only decides a sticky digit
        e10 += len(ds) - 801
        ds = ds[:800] + ("1" if ds[800:].strip("0") else "0")
    if not ds or len(ds) + e10 < -400:
        v = Fraction(0)
    elif len(ds) + e10 > 400:
        return (sign_bit if neg else 0) | inf_bits(bits)
    else:
        v = Fraction(int(ds)) * Fraction(10) ** e10
    return (sign_bit if neg else 0) | round_to_bits(v, bits)


def to_bool(text):
    if text is None:
        return None
    if isinstance(text, bytes):
        text = text.decode("latin-1")
    t = text.strip("".join(chr(c) for c in range(0x21)) + "\x7f")
    low = "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in t)
    if low in ("t", "true", "y", "yes", "1"):
        return True
    if low in ("f", "false", "n", "no", "0"):
        return False
    return None


def bits_value(b, bits):
    """(negative, exact non-negative value) of a finite pattern"""
    mb, bias = FORMATS[bits]
    ef, fr = (b >> mb) & ((1 << (bits - 1 - mb)) - 1), b & ((1 << mb) - 1)
    c, q = (fr | (1 << mb), ef - bias - mb) if ef else (fr, 1 - bias - mb)
    return bool(b >> (bits - 1)), Fraction(c) * Fraction(2) ** q


def _interval(b, bits):
    """the rounding interval of the positive finite pattern b: (low, high, closed)"""
    mb, _ = FORMATS[bits]
    _, v = bits_value(b, bits)
    _, up = bits_value(b + 1, bits)
    lo = bits_value(b - 1, bits)[1] if b > 1 else Fraction(0)
    return (lo + v) / 2 if b > 0 else Fraction(0), (v + up) / 2, (b & ((1 << mb) - 1)) % 2 == 0


def float_to_text(b, bits):
    mb, _ = FORMATS[bits]
    emask = (1 << (bits - 1 - mb)) - 1
    neg = bool(b >> (bits - 1))
    ab = b & ((1 << (bits - 1)) - 1)
    if ab >> mb == emask:
        return "NaN" if ab & ((1 << mb) - 1) else ("-Infinity" if neg else "Infinity")
    if ab == 0:
        return "-0.0" if neg else "0.0"
    _, x = bits_value(ab, bits)
    lo, hi, closed = _interval(ab, bits)

    def inside(d):
        return lo <= d <= hi if closed else lo < d < hi

    e = len(str(x.numerator)) - len(str(x.denominator))   # 10^e <= x < 10^(e + 1)
    while Fraction(10) ** e > x:
        e -= 1
    while Fraction(10) ** (e + 1) <= x:
        e += 1

    def nearest(length):   # the decimals of at most `length` digits just below and just above x
        g = Fraction(10) ** (e - length + 1)
        n = x / g
        dn = n.numerator // n.denominator
        return [(dn, g), (dn + 1, g)] if dn * g != x else [(dn, g)]

    m = next(L for L in range(1, 20) if any(inside(n * g) for n, g in nearest(L)))
    cands = [(n, g) for n, g in nearest(max(m, 2)) if inside(n * g)]
    n, g = min(cands, key=lambda ng: (abs(ng[0] * ng[1] - x), ng[0] % 2))
    # n * g as digits and the exponent of the first digit
    s = str(n).rstrip("0")
    p = 0   # g = 10^p
    gg = g
    while gg.denominator != 1:
        gg *= 10
        p -= 1
    while gg.numerator != 1:
        gg /= 10
        p += 1
    exp10 = len(str(n)) - 1 + p
    if -3 <= exp10 < 7:
        if exp10 >= 0:
            ip = s[:exp10 + 1].ljust(exp10 + 1, "0")
            fp = s[exp10 + 1:] or "0"
        else:
            ip, fp = "0", "0" * (-exp10 - 1) + s
        out = f"{ip}.{fp}"
    else:
        out = f"{s[0]}.{s[1:] or '0'}E{exp10}"
    return ("-" if neg else "") + out


def decimal_to_text(unscaled, scale):
    if unscaled is None:
        return None
    digits = str(abs(unscaled))
    if scale > 0:
        digits = digits.rjust(scale + 1, "0")
        digits = digits[:-scale] + "." + digits[-scale:]
    return ("-" if unscaled < 0 else "") + digits
