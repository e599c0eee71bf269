"""CPU checks of tests/expr_reference.py: hand-computed values and the reference's own unit-test vectors (paths relative to
native-engine/).  The GPU edge tests trust this file, so it is pinned here first."""
import datetime as dt
import math

import expr_reference as R
from key_reference import f32_bits, f64_bits

NAN64 = 0x7FF8000000000000


def test_integer_arithmetic_wraps_per_width():
    assert R.arith("Plus", 127, 1, "int8") == -128
    assert R.arith("Minus", -32768, 1, "int16") == 32767
    assert R.arith("Multiply", 2**31 - 1, 2, "int32") == -2
    assert R.arith("Multiply", -2**63, -1, "int64") == -2**63
    assert R.arith("Divide", -128, -1, "int8") == -128                       # MIN / -1 wraps
    assert R.arith("Divide", -2**63, -1, "int64") == -2**63
    assert R.arith("Modulo", -2**63, -1, "int64") == 0
    assert R.arith("Divide", -7, 2, "int32") == -3                           # truncates toward zero
    assert R.arith("Modulo", -7, 2, "int32") == -1                           # sign of the dividend
    assert R.arith("Modulo", 7, -2, "int32") == 1
    assert R.arith("Divide", 5, 0, "int32") is None and R.arith("Modulo", 5, 0, "int64") is None
    assert R.arith("Plus", None, 1, "int32") is None


def test_bitwise_and_shifts_mask_the_count():
    assert R.arith("BitwiseShiftLeft", 1, 33, "int32") == 2                  # 33 & 31
    assert R.arith("BitwiseShiftLeft", 1, 65, "int64") == 2                  # 65 & 63
    assert R.arith("BitwiseShiftLeft", 1, 31, "int32") == -2**31
    assert R.arith("BitwiseShiftLeft", 1, 7, "int8") == -128                 # wraps to the int8 width
    assert R.arith("BitwiseShiftLeft", 1, 8, "int8") == 0
    assert R.arith("BitwiseShiftRight", -8, 1, "int32") == -4                # arithmetic shift
    assert R.arith("BitwiseShiftRight", -1, 63, "int64") == -1
    assert R.arith("BitwiseAnd", -1, 0x55, "int16") == 0x55
    assert R.arith("BitwiseXor", -1, 0, "int64") == -1
    assert R.arith("BitwiseOr", -128, 127, "int8") == -1


def test_float_arithmetic_rounds_once_to_its_type():
    one = f32_bits(1.0)
    tiny = f32_bits(2.0 ** -24)                                              # half an ulp of 1.0f: ties to even
    assert R.arith("Plus", one, tiny, "float32") == one
    assert R.arith("Plus", one, f32_bits(3 * 2.0 ** -25), "float32") == f32_bits(1.0 + 2.0 ** -23)
    assert R.arith("Divide", one, 0, "float32") == f32_bits(math.inf)
    assert R.arith("Divide", one, 1 << 31, "float32") == f32_bits(-math.inf)   # 1 / -0.0
    assert math.isnan(R.to_float(R.arith("Divide", 0, 0, "float64"), "float64"))
    assert R.arith("Multiply", f64_bits(1e308), f64_bits(10.0), "float64") == f64_bits(math.inf)
    assert R.arith("Modulo", f64_bits(-7.5), f64_bits(2.0), "float64") == f64_bits(-1.5)
    assert R.negate(0, "float64") == 1 << 63                                # -0.0
    assert R.negate(-128, "int8") == -128


def test_compare_total_order_and_kleene():
    nan, neg0 = NAN64, 1 << 63
    assert R.compare("Eq", nan, nan, "float64") is True
    assert R.compare("Lt", neg0, 0, "float64") is True                      # -0.0 < +0.0
    assert R.compare("Gt", nan, f64_bits(math.inf), "float64") is True
    assert R.compare("Lt", None, 1, "int32") is None
    assert R.compare("IsNotDistinctFrom", None, None, "int32") is True
    assert R.compare("IsNotDistinctFrom", None, 1, "int32") is False
    assert [R.kleene_and(a, b) for a, b in [(True, None), (False, None), (None, None), (True, True)]] == [None, False, None, True]
    assert [R.kleene_or(a, b) for a, b in [(True, None), (False, None), (None, None), (False, False)]] == [True, None, None, False]


def test_casts_hand_values():
    assert R.cast(300, "int32", "int8") is None and R.cast(-128, "int64", "int8") == -128
    assert R.cast(f64_bits(math.nan), "float64", "int32") == 0
    assert R.cast(f64_bits(3e9), "float64", "int32") == 2**31 - 1
    assert R.cast(f64_bits(-1e30), "float64", "int64") == -2**63
    assert R.cast(f64_bits(-2.9), "float64", "int16") == -2
    assert R.cast(f64_bits(0.125), "float64", ("dec", 9, 2)) == 13            # 12.5 -> 13: half away from zero
    assert R.cast(f64_bits(-0.125), "float64", ("dec", 9, 2)) == -13
    assert R.cast(f64_bits(2.5), "float64", ("dec", 9, 0)) == 3                # Python's round(2.5) would be 2
    assert R.cast(f64_bits(1e10), "float64", ("dec", 9, 0)) is None
    assert R.cast(12345, ("dec", 10, 3), ("dec", 7, 2)) == 1235
    assert R.cast(-12345, ("dec", 10, 3), ("dec", 7, 2)) == -1235
    assert R.cast(-12355, ("dec", 10, 3), ("dec", 7, 1)) == -124
    assert R.cast(-7999, ("dec", 10, 3), "int32") == -7                        # truncates
    assert R.cast(10**20, ("dec", 38, 0), "int64") is None
    assert R.cast(-5, ("dec", 10, 1), "float64") == f64_bits(-0.5)
    # decimal -> float rounds once: 2^117 + 2^64 + 2^63 lies 3/4 of an ulp above 2^117
    v = ((2**53 + 1) << 64) + 2**63
    assert R.cast(v, ("dec", 38, 0), "float64") == f64_bits(2.0 ** 117 + 2.0 ** 65)
    assert R.cast(True, "bool", "int32") == 1 and R.cast(2, "int8", "bool") is True


def test_check_overflow_golden():
    # datafusion-ext-functions/src/spark_check_overflow.rs:137-160: (20, 8) -> (10, 5)
    vals = [12342132145623, 13245, 123213244568923, 1234567890, None]
    assert [R.check_overflow(v, 8, 10, 5) for v in vals] == [None, 13, None, 1234568, None]
    assert R.check_overflow(10**10, 2, 10, 2) is None                         # same type: re-checked (Spark)
    assert R.check_overflow(-5, 1, 10, 0) == -1 and R.check_overflow(5, 1, 10, 0) == 1


def test_make_decimal_and_unscaled_goldens():
    # spark_make_decimal.rs:74-100 passes every value through; Spark (and this engine) give NULL past the precision
    vals = [12342132145623, 13245, 123213244568923, 1234567890, None]
    assert [R.make_decimal(v, 10, null_on_overflow=False) for v in vals] == vals
    assert [R.make_decimal(v, 10) for v in vals] == [None, 13245, None, 1234567890, None]
    # spark_unscaled_value.rs
    assert [R.unscaled_value(v) for v in [1234567890987654321, 9876543210, 135792468109, None, 67898]] == \
        [1234567890987654321, 9876543210, 135792468109, None, 67898]
    assert R.unscaled_value(2**64 + 5) == 5 and R.unscaled_value(2**63) == -2**63 and R.unscaled_value(-(2**64) - 1) == -1


def test_null_if_goldens():
    # spark_null_if.rs: NullIfZero
    assert [R.null_if_zero(v, "int32") for v in [1, None, -1, 0]] == [1, None, -1, None]
    assert R.null_if_zero(1230427389124691, "dec") == 1230427389124691
    assert R.null_if_zero(f32_bits(0.0), "float32") is None and R.null_if_zero(f32_bits(-0.0), "float32") is None
    assert [R.null_if(a, b) for a, b in [(1, 1), (1, 2), (None, 1), (1, None)]] == [None, 1, None, 1]
    assert R.coalesce(None, None, 3, 4) == 3 and R.coalesce(None) is None
    assert R.normalize_nan_and_zero(f64_bits(-0.0), "float64") == 0
    assert R.normalize_nan_and_zero(0xFFF8000000000123, "float64") == NAN64


def test_spark_decimal_result_types():
    assert R.adjust_precision_scale(49, 2) == (38, 2)
    assert R.adjust_precision_scale(77, 20) == (38, 6)
    assert R.adjust_precision_scale(39, 2) == (38, 2)
    assert R.adjust_precision_scale(39, 10) == (38, 9)
    assert R.result_decimal_type("Multiply", 38, 2, 10, 0) == (38, 2)
    assert R.result_decimal_type("Multiply", 9, 2, 7, 4) == (17, 6)
    assert R.result_decimal_type("Plus", 38, 2, 38, 2) == (38, 2)
    assert R.result_decimal_type("Minus", 18, 0, 18, 0) == (19, 0)
    assert R.result_decimal_type("Multiply", 38, 10, 38, 10) == (38, 6)
    assert R.engine_arith_type("Multiply", 38, 2, 10, 0) == (38, 2)
    assert R.engine_arith_type("Plus", 9, 2, 18, 2) == (19, 2)
    assert R.engine_arith_type("Plus", 9, 2, 10, 4) == (12, 4)                 # (9, 2) is brought to (11, 4) first


def test_decimal_arithmetic_overflow_gives_null():
    # (38,2) x (10,0): 6e37 * 2 has 39 digits; 1e37 * 50 passes 2^127
    assert R.spark_decimal_op("Multiply", 6 * 10**37, 38, 2, 2, 10, 0) is None
    assert R.spark_decimal_op("Multiply", 10**37, 38, 2, 50, 10, 0) is None
    assert R.spark_decimal_op("Multiply", 5 * 10**36, 38, 2, 2, 10, 0) == 10**37
    m = 10**38 - 1
    assert R.spark_decimal_op("Plus", m, 38, 2, m, 38, 2) is None
    assert R.spark_decimal_op("Plus", m, 38, 2, -m, 38, 2) == 0
    assert R.spark_decimal_op("Minus", -(10**18 - 1), 18, 0, 10**18 - 1, 18, 0) == -(2 * 10**18 - 2)
    # (9,2) x (7,4) at (17,6): 1.23 * 0.0005 = 0.000615 and -0.01 * 0.0005 = -0.000005, both exact
    assert R.spark_decimal_op("Multiply", 123, 9, 2, 5, 7, 4) == 615
    assert R.spark_decimal_op("Multiply", -1, 9, 2, 5, 7, 4) == -5
    # (38,10) x (38,10) at (38,6): lhs is rounded to scale 6 first, the product rounds from scale 16 to 6
    assert R.spark_decimal_op("Multiply", 15000, 38, 10, 10**10, 38, 10) == 2    # 0.0000015 -> 0.000002 (half away), x 1
    assert R.decimal_binary("Plus", 1, 2, 1, 4, 12) == 101


def test_round_half_up_and_even():
    assert R.round_decimal(12345, 2, 1) == 12350 and R.round_decimal(-67895, 2, 1) == -67900
    assert R.round_decimal(12345, 2, 1, half_even=True) == 12340 and R.round_decimal(67895, 2, 1, half_even=True) == 67900
    assert R.round_int(314159265, -2) == 314159300 and R.round_int(-25, -1) == -30 and R.round_int(-25, -1, True) == -20
    assert R.round_int(-2**63, -1) == 2**63 - 2 and R.round_int(2**31 - 1, -1, bits=32) == -2**31 + 2    # i128 result truncated


def test_dates_against_python():
    epoch = dt.date(1970, 1, 1)
    for d in [-719162, -719163, -1, 0, 1, 59, 10957, 11016, 18321, 19000, 2932896, 2932897]:
        if -719162 <= d <= 2932896:
            x = epoch + dt.timedelta(days=d)
            assert R.civil_from_days(d) == (x.year, x.month, x.day)
            assert R.days_from_civil(x.year, x.month, x.day) == d
            assert R.date_part(d, "dayofweek") == x.isoweekday() % 7 + 1
            assert R.date_part(d, "dow") == x.isoweekday() % 7                 # Sunday = 0
            assert R.date_part(d, "week") == x.isocalendar()[1]
            assert R.date_part(d, "doy") == x.timetuple().tm_yday
            assert R.date_text(d) == x.isoformat().encode()
    assert R.date_text(-719163) == b"0000-12-31"
    assert R.date_text(-719528) == b"0000-01-01"
    assert R.date_text(-719529) == b"-0001-12-31"
    assert R.date_text(2932897) == b"+10000-01-01"                            # chrono: {:+05} outside 0..9999
    assert R.date_text(-(2**31)) == b"-5877641-06-23" and R.date_text(2**31 - 1) == b"+5881580-07-11"


def test_strings():
    assert R.trim(b"  a b \t ") == b"a b \t" and R.trim(b"  a ", "left") == b"a " and R.trim(b"  a ", "right") == b"  a"
    assert R.ascii_upper("aé z".encode()) == "Aé Z".encode() and R.ascii_lower(b"AbC") == b"abc"
    assert R.octet_length("é".encode()) == 2
    assert R.decimal_text(-5, 3) == b"-0.005" and R.decimal_text(123, 0) == b"123" and R.decimal_text(0, 2) == b"0.00"
