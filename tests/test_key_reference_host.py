"""CPU checks of tests/key_reference.py, the plain-Python reference that test_gpu_key_edges.py holds the kernels to."""
import math

import pytest

import key_reference as R
from key_reference import bits_f32, bits_f64, f32_bits, f64_bits


def _sorted(vals, t, asc=True, nulls_first=True):
    return sorted(vals, key=lambda v: R.sort_key(v, t, asc, nulls_first))


@pytest.mark.parametrize("t,width", [("float32", 32), ("float64", 64)])
def test_float_ladder_is_ieee_total_order(t, width):
    sign = 1 << (width - 1)
    fb = f32_bits if t == "float32" else f64_bits
    inf = fb(math.inf)
    quiet = inf | (1 << (22 if width == 32 else 51))
    ladder = [sign | quiet | 1, sign | quiet, sign | inf, fb(-3.5), fb(-1.0), sign | 1, sign, 0, 1, fb(1.0), fb(3.5), inf - 1, inf,
              quiet, quiet | 1, quiet | 0x2345]
    shuffled = ladder[::2] + ladder[1::2]
    assert _sorted(shuffled, t) == ladder
    assert _sorted(shuffled + [None], t, nulls_first=False) == ladder + [None]
    assert _sorted(shuffled + [None], t, asc=False, nulls_first=True) == [None] + ladder[::-1]
    assert set(R.edge_values(t)) <= set(ladder) | {R.SENTINEL}


def test_float64_sentinel_bits_are_a_negative_number():
    assert R.SENTINEL >> 63 == 1
    v = bits_f64(R.SENTINEL)
    assert v < 0 and not math.isnan(v)
    assert R.total_order(f64_bits(-1.0), 64) < R.total_order(R.SENTINEL, 64) < R.total_order(f64_bits(-0.0), 64)


def test_decimal_ladder_orders_as_exact_integers():
    w = 1 << 64
    ladder = [-(10 ** 38 - 1), -w - 1, -w, -(w - 1), -5, -1, 0, 1, 5, w - 1, w, w + 1, 2 * w + 1, 10 ** 38 - 1]
    assert _sorted(ladder[::-1], "dec38_10") == ladder
    assert _sorted(ladder, "dec38_10", asc=False) == ladder[::-1]
    # the values that share a low word: 1, 1 + 2^64, 1 + 2^65, 1 - 2^64
    lows = {v & (w - 1) for v in (1, 1 + w, 1 + 2 * w, 1 - w)}
    assert lows == {1}
    assert {1 + w, 1 + 2 * w, 1 - w} <= set(R.edge_values("dec38_10"))


def test_string_ladder_is_unsigned_bytewise_with_shorter_prefix_first():
    ladder = [b"", b"\x00", b"\x00\x00", b"a", b"a\x00", b"ab", b"a\x7f", b"a\x80", b"a\xff", b"q" * 7 + b"a", b"q" * 7 + b"b",
              b"q" * 8 + b"a", "é".encode(), "ÿ".encode(), "\U0001F600".encode(), b"\xff", b"\xff" * 8, b"\xff" * 9]
    assert _sorted(ladder[::-1], "binary") == ladder
    assert _sorted(ladder + [None], "utf8", asc=False, nulls_first=False) == ladder[::-1] + [None]
    assert R.sort_key(b"a", "utf8") < R.sort_key(b"a\x00", "utf8")


def test_narrow_types_and_multi_key_order():
    assert _sorted([True, None, False], "bool") == [None, False, True]
    assert _sorted([127, -128, 0, None], "int8", asc=False, nulls_first=False) == [127, 0, -128, None]
    specs = [("int8", True, False), ("utf8", False, True)]
    rows = [(1, b"a"), (None, b"b"), (1, None), (-1, b"z"), (1, b"b")]
    assert sorted(rows, key=lambda r: R.row_sort_key(r, specs)) == [(-1, b"z"), (1, None), (1, b"b"), (1, b"a"), (None, b"b")]


def test_reference_float_equality_statements_hold_for_ieee_eq():
    # datafusion-ext-commons/src/arrow/eq_comparator.rs:443-474: the reference's hash joins compare floats with `==`, where NaN is
    # not equal to NaN and -0.0 equals 0.0.  The engine deliberately compares bits instead (DESIGN section 4); these are the
    # statements it differs from.
    nan, neg0 = float("nan"), -0.0
    assert not nan == nan
    assert neg0 == 0.0 and f64_bits(neg0) != f64_bits(0.0)
    assert bits_f32(f32_bits(neg0)) == 0.0
    # the engine's join reference: bitwise
    assert R.join_rows([(f64_bits(nan),), (f64_bits(neg0),)], [(f64_bits(nan),), (f64_bits(0.0),)], "INNER") == [(0, 0)]


def test_wrapping_sums_and_div_euclid_match_hand_computed_values():
    mx = (1 << 63) - 1
    assert R.wrapping_sum([mx, mx]) == -2
    assert R.wrapping_sum([-(1 << 63), -1]) == mx
    assert R.wrapping_sum([None, None]) is None
    assert R.wrapping_sum([None, 5, -7]) == -2
    m128 = (1 << 127) - 1
    assert R.wrapping_sum([m128, 1], 128) == -(1 << 127)
    assert R.wrapping_sum([10 ** 38 - 1] * 2, 128) == 2 * 10 ** 38 - 2 - (1 << 128)   # 2 (10^38 - 1) > 2^127 - 1: wraps
    assert R.wrapping_sum([10 ** 37] * 3 + [-(10 ** 37)] * 5, 128) == -2 * 10 ** 37
    assert R.div_euclid(7, 2) == 3 and R.div_euclid(-7, 2) == -4 and R.div_euclid(-8, 2) == -4
    assert R.div_euclid(7, -2) == -3 and R.div_euclid(-7, -2) == 4
    assert R.decimal_avg([-3, None, -4]) == -4                                    # -7 / 2 = -3.5 -> -4 (remainder 1 >= 0)
    assert R.decimal_avg([None]) is None


def test_extremes_use_total_order():
    t = "float64"
    vals = [f64_bits(0.0), f64_bits(-0.0), f64_bits(math.inf), f64_bits(math.nan), None]
    assert R.extreme(vals, t, True) == f64_bits(math.nan)
    assert R.extreme(vals, t, False) == f64_bits(-0.0)
    assert R.extreme([None], t, False) is None
    assert R.extreme([-5, 3, None], "int32", True) == 3


def test_range_partition_is_bisect_left():
    specs = [("float64", True, True)]
    bounds = [(f64_bits(-0.0),), (f64_bits(0.0),), (f64_bits(math.nan),)]
    keys = [(None,), (f64_bits(-1.0),), (f64_bits(-0.0),), (f64_bits(0.0),), (f64_bits(math.inf),), (f64_bits(math.nan),)]
    assert R.range_partition_ids(keys, bounds, specs) == [0, 0, 0, 1, 2, 2]


def test_join_reference_never_matches_null():
    l = [(1,), (None,), (2,), (2,)]
    r = [(2,), (None,), (3,)]
    assert R.join_rows(l, r, "INNER") == [(2, 0), (3, 0)]
    assert R.join_rows(l, r, "FULL") == [(0, None), (1, None), (2, 0), (3, 0), (None, 1), (None, 2)]
    assert R.join_rows(l, r, "ANTI") == [(0, None), (1, None)]
    assert R.join_rows(l, r, "SEMI") == [(2, None), (3, None)]
    assert R.join_rows(l, r, "RIGHT") == [(2, 0), (3, 0), (None, 1), (None, 2)]


@pytest.mark.parametrize("t", R.TYPES)
def test_generator_is_deterministic_and_contains_every_edge(t):
    a = R.edge_column(t, 9000, seed=5)
    assert a == R.edge_column(t, 9000, seed=5)
    assert a != R.edge_column(t, 9000, seed=6)
    assert None in a
    assert set(R.edge_values(t)) <= set(a)
    for b in (R.SCAN_BLOCK, R.RADIX_TILE, 2 * R.RADIX_TILE):      # edge values sit on both sides of the block / tile boundaries
        assert {a[b - 1], a[b]} <= set(R.edge_values(t)) | {None}
    assert None not in R.edge_column(t, 100, seed=1, null_rate=0)
    assert set(R.edge_values(t)) <= set(R.edge_column(t, 50, seed=2, null_rate=0))
    assert len(set(R.edge_values(t))) == len(R.edge_values(t))


def test_int_edges_and_sentinel():
    assert R.edge_values("int8") == [-128, -127, -1, 0, 1, 126, 127]
    assert R.SENTINEL_I64 in R.edge_values("int64") and R.SENTINEL_I64 < 0
    assert R.wrap(R.SENTINEL, 64) == R.SENTINEL_I64
    assert R.SENTINEL in R.edge_values("float64")
