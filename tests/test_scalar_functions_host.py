"""CPU checks of greatest, least, nvl2, months_between, date_trunc, make_date, hex, chr, acosh, factorial, RowNum and
spark_partition_id: the plain-Python reference (scalar_reference.py) against the reference's months_between goldens and
hand-computed values, and the planner, through runtime.explain, accepting every supported position and naming the function in
every rejected one."""
import datetime as dt
from zoneinfo import ZoneInfo

import pyarrow as pa
import pytest

import scalar_reference as R
from auron_b200 import proto as P
from auron_b200 import runtime


def utc_ms(y, mo, d, h=0, mi=0, s=0):
    return int(dt.datetime(y, mo, d, h, mi, s, tzinfo=dt.timezone.utc).timestamp()) * 1000


# ------------------------------------------------------------------------------------------------------------ reference
def test_months_between_goldens():
    # spark_dates.rs:953-1074
    assert R.months_between(utc_ms(2024, 3, 15, 23, 59, 59), utc_ms(2024, 1, 15), True, "UTC") == 2.0
    assert R.months_between(utc_ms(2024, 2, 29, 12), utc_ms(2024, 1, 31), True, "UTC") == 1.0
    assert R.months_between(utc_ms(2024, 3, 2, 12), utc_ms(2024, 1, 1), True, "UTC") == 2.0483871
    assert abs(R.months_between(utc_ms(2024, 3, 2, 12), utc_ms(2024, 1, 1), False, "UTC") - 2.0483870967741935) < 1e-12
    assert abs(R.months_between(utc_ms(2024, 3, 10, 7, 30), utc_ms(2024, 2, 9, 6, 30), False, "America/New_York") - 1.0336021505376345) < 1e-12
    assert R.months_between(utc_ms(2024, 1, 15), utc_ms(2024, 3, 15, 23, 59, 59), True, "UTC") == -2.0
    assert R.months_between(utc_ms(2024, 1, 1), utc_ms(2024, 3, 2, 12), True, "UTC") == -2.0483871
    assert R.months_between(None, utc_ms(2024, 1, 1), True, "UTC") is None


def test_months_between_rules():
    assert R.months_between(utc_ms(2024, 3, 2, 12), utc_ms(2024, 1, 1), True, None) == 2.0483871   # no zone: UTC
    assert R.months_between(utc_ms(2024, 3, 2, 12), utc_ms(2024, 1, 1), True, "Not/AZone") == 2.0483871
    assert R.months_between(utc_ms(2024, 3, 2), utc_ms(2024, 1, 1), None, "UTC") is None
    # before 1970; the seconds of a day before the epoch still count from that day's midnight
    assert R.months_between(utc_ms(1969, 12, 31, 6), utc_ms(1969, 11, 30, 18), False, None) == 1.0   # both on the last day
    assert R.months_between(utc_ms(1969, 12, 30, 6), utc_ms(1969, 11, 29, 18), False, None) == 1 + (86400 + 6 * 3600 - 18 * 3600) / 2678400
    # a result that rounds to a negative value: (-86400 - 1) / 2678400 = -0.0322584378...
    assert R.months_between(utc_ms(2024, 1, 1), utc_ms(2024, 1, 2, 0, 0, 1), True, None) == -0.03225844
    assert R.to_ms(-1, "us") == 0 and R.to_ms(-1999, "us") == -1 and R.to_ms(3, "date32") == 3 * 86_400_000 and R.to_ms(-2, "s") == -2000


def test_local_midnight_lookups_against_zoneinfo():
    # America/Sao_Paulo 2018-11-04: DST starts at midnight, so 00:00 does not exist; the first minute that does is 01:00 -02:00
    assert R.start_of_local_day_ms(dt.date(2018, 11, 4), ZoneInfo("America/Sao_Paulo")) == utc_ms(2018, 11, 4, 3)
    # America/Havana 2022-11-06: DST ends at 01:00, so 00:00-00:59 happens twice; the earlier one is 00:00 -04:00
    assert R.start_of_local_day_ms(dt.date(2022, 11, 6), ZoneInfo("America/Havana")) == utc_ms(2022, 11, 6, 4)
    # Australia/Lord_Howe moves by 30 minutes, at 02:00; midnight is ordinary
    assert R.start_of_local_day_ms(dt.date(2023, 10, 1), ZoneInfo("Australia/Lord_Howe")) == utc_ms(2023, 9, 30, 13, 30)
    assert R.start_of_local_day_ms(dt.date(2023, 10, 2), ZoneInfo("Australia/Lord_Howe")) == utc_ms(2023, 10, 1, 13)
    assert R.start_of_local_day_ms(dt.date(2024, 1, 1), ZoneInfo("Asia/Kathmandu")) == utc_ms(2023, 12, 31, 18, 15)
    assert R.local_date(utc_ms(2024, 3, 10, 4, 59), ZoneInfo("America/New_York")) == dt.date(2024, 3, 9)
    assert R.local_date(utc_ms(2024, 3, 10, 5), ZoneInfo("America/New_York")) == dt.date(2024, 3, 10)


def test_date_trunc_every_level():
    us = utc_ms(2024, 8, 14, 13, 47, 25) * 1000 + 123_456   # a Wednesday
    exp = {"YEAR": (2024, 1, 1), "YYYY": (2024, 1, 1), "yy": (2024, 1, 1), "QUARTER": (2024, 7, 1), "month": (2024, 8, 1), "MON": (2024, 8, 1),
           "MM": (2024, 8, 1), "WEEK": (2024, 8, 12), "DAY": (2024, 8, 14), "dd": (2024, 8, 14)}
    for f, ymd in exp.items():
        assert R.date_trunc(f, us, "us") == utc_ms(*ymd) * 1000, f
    assert R.date_trunc("HOUR", us, "us") == utc_ms(2024, 8, 14, 13) * 1000
    assert R.date_trunc("MINUTE", us, "us") == utc_ms(2024, 8, 14, 13, 47) * 1000
    assert R.date_trunc("SECOND", us, "us") == utc_ms(2024, 8, 14, 13, 47, 25) * 1000
    assert R.date_trunc("MILLISECOND", us, "us") == utc_ms(2024, 8, 14, 13, 47, 25) * 1000 + 123_000
    assert R.date_trunc("MICROSECOND", us, "us") == us
    assert R.date_trunc("MICROSECOND", 1_234_567, "ns") == 1_234_000 and R.date_trunc("MILLISECOND", 7, "s") == 7
    # toward -inf before 1970
    assert R.date_trunc("DAY", -1, "us") == -86_400_000_000
    assert R.date_trunc("SECOND", -1, "ms") == -1000
    assert R.date_trunc("WEEK", 0, "s") == -3 * 86400   # 1970-01-01 is a Thursday
    assert R.date_trunc("QUARTER", utc_ms(1969, 12, 31) // 1000, "s") == utc_ms(1969, 10, 1) // 1000
    # unknown / NULL formats, a result below int64, a coarser result unit
    assert R.date_trunc("DECADE", us, "us") is None and R.date_trunc(None, us, "us") is None and R.date_trunc("DAY", None, "us") is None
    assert R.date_trunc("YEAR", -(2**63), "ns") is None
    assert R.date_trunc("DAY", us, "us", "ms") == utc_ms(2024, 8, 14) and R.date_trunc("HOUR", 5, "s", "ns") == 0


def test_make_date_factorial_hex_chr():
    assert R.make_date(1970, 1, 1) == 0 and R.make_date(2024, 2, 29) == 19782 and R.make_date(1969, 12, 31) == -1
    for y, m, d in [(2023, 2, 29), (2024, 0, 1), (2024, 13, 1), (2024, 1, 0), (2024, 1, 32), (2024, 4, 31), (1900, 2, 29)]:
        assert R.make_date(y, m, d) is None, (y, m, d)
    assert R.make_date(2000, 2, 29) == 11016 and R.make_date(-1, 3, 1) == -719468 - 366   # 0000-03-01 is day -719468; year 0 is a leap year
    assert R.make_date(5_881_580, 7, 11) == 2**31 - 1 and R.make_date(5_881_580, 7, 12) is None
    assert R.make_date(-5_877_641, 6, 23) == -(2**31) and R.make_date(-5_877_641, 6, 22) is None
    assert R.make_date(None, 1, 1) is None
    assert [R.factorial(n) for n in (-1, 0, 1, 5, 20, 21, None)] == [None, 1, 1, 120, 2432902008176640000, None, None]
    assert R.hex_int(0) == b"0" and R.hex_int(-1) == b"F" * 16 and R.hex_int(255) == b"FF" and R.hex_int(-(2**63)) == b"8" + b"0" * 15
    assert R.hex_int(2**63 - 1) == b"7" + b"F" * 15 and R.hex_int(None) is None
    assert R.hex_bytes(b"") == b"" and R.hex_bytes(b"\x00\xffA") == b"00FF41" and R.hex_bytes("é".encode()) == b"C3A9"
    assert R.chr_(-1) == b"" and R.chr_(0) == b"\x00" and R.chr_(65) == b"A" and R.chr_(127) == b"\x7f"
    assert R.chr_(128) == b"\xc2\x80" and R.chr_(255) == "ÿ".encode() and R.chr_(256 + 65) == b"A" and R.chr_(-(2**63)) == b""


def test_greatest_least_order():
    nan, inf = float("nan"), float("inf")
    assert R.greatest([1.0, nan, inf], "f64") is nan and R.greatest([1.0, nan, -inf], "f64", least=True) == -inf
    assert str(R.greatest([-0.0, 0.0], "f64")) == "0.0" and str(R.greatest([0.0, -0.0], "f64", least=True)) == "-0.0"
    assert R.greatest([None, None], "int") is None and R.greatest([None, 3, None, 5], "int") == 5
    assert R.greatest([b"ab", b"ab\x00", b"a\xff"], "bytes") == b"a\xff" and R.greatest([b"ab", b"ab\x00"], "bytes", least=True) == b"ab"
    assert R.nvl2(None, 1, 2) == 2 and R.nvl2(0, 1, 2) == 1 and R.nvl2(0, None, 2) is None


# ------------------------------------------------------------------------------------------------------------ planning
SCHEMA = pa.schema([("s", pa.string()), ("t", pa.string()), ("b", pa.binary()), ("i", pa.int64()), ("j", pa.int64()), ("n", pa.int32()),
                    ("m", pa.int32()), ("f", pa.float64()), ("g", pa.float64()), ("d", pa.decimal128(38, 2)), ("e", pa.decimal128(38, 2)),
                    ("ts", pa.timestamp("us")), ("tn", pa.timestamp("ns")), ("dt", pa.date32()), ("bo", pa.bool_()), ("r", pa.bool_())])
U, I32, I64, F64, D32 = pa.string(), pa.int32(), pa.int64(), pa.float64(), pa.date32()
TS = pa.timestamp("us")


def _fn(name, *args, t=U):
    return P.scalar_fn(name, list(args), t)


def _lit(v, t=U):
    return P.lit(v, t)


def _explain(plan, partition_id=0):
    return runtime.explain(P.task_definition(plan, partition_id=partition_id))


def _src():
    return P.ffi_reader(SCHEMA, "t")


def _project(exprs, types, src=None):
    return P.projection(src or _src(), exprs, [f"c{i}" for i in range(len(exprs))], types)


c = P.col
VALUES = {   # name -> (expression, type): valid anywhere
    "greatest_i64": (_fn("Greatest", c("i"), c("j"), _lit(None, I64), t=I64), I64),
    "least_f64": (_fn("Least", c("f"), c("g"), t=F64), F64),
    "greatest_dec": (_fn("Greatest", c("d"), c("e"), t=pa.decimal128(38, 2)), pa.decimal128(38, 2)),
    "least_utf8": (_fn("Least", c("s"), c("t"), _lit("m"), t=U), U),
    "greatest_binary": (_fn("Greatest", c("b"), _lit(b"x", pa.binary()), t=pa.binary()), pa.binary()),
    "greatest_ts": (_fn("Greatest", c("ts"), _lit(0, TS), t=TS), TS),
    "least_bool": (_fn("Least", c("bo"), c("r"), t=pa.bool_()), pa.bool_()),
    "greatest_12": (_fn("Greatest", *[P.binary("Plus", c("i"), _lit(k, I64)) for k in range(12)], t=I64), I64),
    "nvl2_utf8": (_fn("Nvl2", c("i"), c("s"), _fn("Upper", c("t")), t=U), U),
    "nvl2_null_then": (_fn("Nvl2", c("s"), _lit(None, pa.null()), c("n"), t=I32), I32),
    "months_between": (_fn("Spark_MonthsBetween", c("ts"), c("dt"), c("r"), _lit("America/New_York"), t=F64), F64),
    "months_between_ns_utc": (_fn("Spark_MonthsBetween", c("tn"), c("ts"), _lit(True, pa.bool_()), _lit(None), t=F64), F64),
    "date_trunc": (_fn("DateTrunc", _lit("month"), c("ts"), t=TS), TS),
    "date_trunc_ns": (_fn("DateTrunc", _lit("YYYY"), c("tn"), t=TS), TS),
    "date_trunc_unknown": (_fn("DateTrunc", _lit("decade"), c("ts"), t=TS), TS),
    "make_date": (_fn("MakeDate", c("n"), c("m"), _lit(1, I32), t=D32), D32),
    "acosh": (_fn("Acosh", c("f"), t=F64), F64),
    "factorial": (_fn("Factorial", c("n"), t=I64), I64),
    "partition_id": (P.spark_partition_id(), I32),
}
BUILDERS = {   # valid as a whole expression, a concat / concat_ws piece and a digest argument
    "hex_int": _fn("Hex", c("i")),
    "hex_int32": _fn("Hex", c("n")),
    "hex_utf8": _fn("Hex", _fn("Upper", c("s"))),
    "hex_binary": _fn("Hex", c("b")),
    "chr": _fn("Chr", c("i")),
    "chr_of_greatest": _fn("Chr", _fn("Greatest", c("i"), c("j"), t=I64)),
}


@pytest.mark.parametrize("name", sorted(VALUES))
def test_value_functions_plan_anywhere(name):
    e, t = VALUES[name]
    plan = _explain(_project([e], [t]))["plan"]
    assert plan["op"] == "ProjectExec"
    probe = P.is_not_null(e)
    _explain(P.filter_(_src(), [probe]))
    _explain(_project([P.case([(P.binary("Gt", c("i"), _lit(0, I64)), e)], None)], [t]))
    _explain(P.agg(_src(), [e], ["k"], [P.agg_expr("COUNT", [c("i")], I64)], ["c"], ["PARTIAL"]))
    _explain(P.sort(_src(), [P.sort_expr(e)]))
    _explain(P.shuffle_writer(_src(), P.hash_repartition([e], 4), "/tmp/x.data", "/tmp/x.index"))


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_hex_and_chr_plan_as_expression_piece_and_digest_argument(name):
    e = BUILDERS[name]
    exprs = [e, _fn("Spark_StringConcat", _lit("<"), e, c("s")), _fn("Spark_StringConcatWs", _lit("|"), c("s"), e, _lit(None)),
             _fn("Spark_MD5", e), _fn("Spark_Sha256", P.try_cast(e, U)), P.try_cast(e, U)]
    plan = _explain(_project(exprs, [U] * len(exprs)))["plan"]
    assert [x[1] for x in plan["schema"]] == ["utf8"] * len(exprs)


def test_row_num_plans_in_a_projection():
    plan = _explain(_project([P.row_num(), P.binary("Plus", P.row_num(), c("i")), _fn("Hex", P.row_num())], [I64, I64, U],
                             src=P.filter_(_src(), [P.binary("Gt", c("i"), _lit(0, I64))])))["plan"]
    assert [x[1] for x in plan["schema"]] == ["int64", "int64", "utf8"]
    assert "RowNum()" in str(plan)
    # the first CASE condition and a non-short-circuit function see every row
    _explain(_project([P.case([(P.binary("Gt", P.row_num(), _lit(3, I64)), _lit(1, I64))], _lit(0, I64)),
                       _fn("Nvl2", c("s"), P.row_num(), _lit(0, I64), t=I64)], [I64, I64]))


def test_spark_partition_id_is_the_task_partition():
    for pid in (0, 7):
        plan = _explain(_project([P.spark_partition_id()], [I32]), partition_id=pid)["plan"]
        assert f"lit(int32:{pid})" in str(plan), plan


REJECTED = {
    "hex_in_comparison": ("Hex", P.binary("Eq", _fn("Hex", c("i")), _lit("x"))),
    "chr_in_case": ("Chr", P.case([(P.is_null(c("s")), _fn("Chr", c("i")))], c("s"))),
    "upper_of_hex": ("Hex", _fn("Upper", _fn("Hex", c("s")))),
    "hex_of_hex": ("Hex", _fn("Hex", _fn("Hex", c("s")))),
    "repeat_of_chr": ("Chr", _fn("Spark_StringRepeat", _fn("Chr", c("i")), _lit(2, I32))),
    "hex_float": ("Hex", _fn("Hex", c("f"))),
    "chr_utf8": ("Chr", _fn("Chr", c("s"))),
    "date_trunc_column_format": ("date_trunc", _fn("DateTrunc", c("s"), c("ts"), t=TS)),
    "date_trunc_date": ("date_trunc", _fn("DateTrunc", _lit("month"), c("dt"), t=TS)),
    "greatest_mixed_types": ("Greatest", _fn("Greatest", c("s"), c("i"), t=U)),
    "least_one_argument": ("Least", _fn("Least", c("i"), t=I64)),
    "factorial_float": ("factorial", _fn("Factorial", c("f"), t=I64)),
    "row_num_in_case_branch": ("RowNum", P.case([(P.is_null(c("s")), P.row_num())], _lit(0, I64))),
    "row_num_in_coalesce": ("RowNum", _fn("Coalesce", c("i"), P.row_num(), t=I64)),
    "row_num_in_sc_and": ("RowNum", P.sc_and(c("bo"), P.binary("Gt", P.row_num(), _lit(1, I64)))),
}


@pytest.mark.parametrize("shape", sorted(REJECTED))
def test_rejected_positions_name_the_function(shape):
    name, expr = REJECTED[shape]
    with pytest.raises(runtime.AuronError, match=name):
        _explain(_project([expr], [U]))


@pytest.mark.parametrize("name", ["Hex", "Chr"])
def test_hex_and_chr_in_a_filter_are_rejected(name):
    with pytest.raises(runtime.AuronError, match=name):
        _explain(P.filter_(_src(), [P.binary("Eq", _fn(name, c("i")), _lit("A"))]))


def test_row_num_outside_a_projection_is_rejected():
    with pytest.raises(runtime.AuronError, match="RowNum"):
        _explain(P.filter_(_src(), [P.binary("Gt", P.row_num(), _lit(3, I64))]))
    with pytest.raises(runtime.AuronError, match="RowNum"):
        _explain(P.agg(_src(), [P.row_num()], ["k"], [P.agg_expr("COUNT", [c("i")], I64)], ["c"], ["PARTIAL"]))


def test_levenshtein_still_names_itself():
    with pytest.raises(runtime.AuronError, match="Levenshtein"):
        _explain(_project([_fn("Levenshtein", c("s"), c("t"), t=I32)], [I32]))
