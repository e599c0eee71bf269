"""CPU checks of lpad, rpad, replace, translate, reverse, initcap, ascii, bit_length, find_in_set and trim with a character set:
the plain-Python reference (string_reference.py) against the reference's initcap goldens and hand-computed values, and the
planner, through runtime.explain, accepting every supported position and naming the function in every rejected one."""
import pyarrow as pa
import pytest

import string_reference as R
from auron_b200 import proto as P
from auron_b200 import runtime

E2, E3, E4 = "é".encode(), "天".encode(), "😁".encode()


# ------------------------------------------------------------------------------------------------------------ reference
def test_initcap_reference_goldens():
    # spark_initcap.rs:80-118
    cases = [(None, None), ("", ""), ("hI THOmAS", "Hi Thomas"), ("James-Smith", "James-smith"), ("michael rose", "Michael Rose"),
             ("a1b2   c3D4", "A1b2   C3d4"), (" ---abc--- ABC --ABC-- a-b A B eB Ac c d", " ---abc--- Abc --abc-- A-b A B Eb Ac C D"),
             (" 世  界  世界 ", " 世  界  世界 "), ("abC c3D4", "Abc C3d4")]
    for s, exp in cases:
        assert R.initcap(None if s is None else s.encode()) == (None if exp is None else exp.encode()), s


def test_initcap_leaves_non_ascii_alone():
    assert R.initcap("éCOLE ßAB ñu".encode()) == "école ßab ñu".encode()   # a non-ASCII character is no separator
    assert R.initcap(b"1st 2ND") == b"1st 2nd"


def test_pad_rules():
    assert R.lpad(b"abc", 5, b"xy") == b"xyabc"
    assert R.rpad(b"abc", 6, b"xy") == b"abcxyx"
    assert R.lpad(b"abcdef", 3, b"x") == b"abc"          # truncates to n characters
    assert R.rpad(b"abcdef", 3, b"x") == b"abc"
    assert R.lpad(b"abc", 10, b"") == b"abc"              # an empty pad returns s
    assert R.lpad(b"abc", 2, b"") == b"ab"                # ... after truncation
    assert R.lpad(b"abc", 0, b"x") == b"" and R.rpad(b"abc", -5, b"x") == b""
    assert R.lpad(b"", 3, b"ab") == b"aba"
    assert R.lpad(E3 * 3, 2, b"x") == E3 * 2              # characters, not bytes
    assert R.lpad(b"a", 4, E2 + E4) == E2 + E4 + E2 + b"a"
    assert R.rpad(E4, 3, E3) == E4 + E3 + E3
    assert R.lpad(b"7", 10, b"0") == b"0000000007"
    assert R.lpad(None, 3, b"x") is None and R.lpad(b"a", None, b"x") is None and R.rpad(b"a", 3, None) is None
    assert R.pad_len(b"ab", 2**63 - 1, b"xyz") == 2 + 3 * ((2**63 - 3) // 3) + (2**63 - 3) % 3
    assert R.pad_len(E2 * 4, 6, E4) == 8 + 8


def test_replace_rules():
    assert R.replace(b"aaa", b"aa", b"b") == b"ba"        # non-overlapping, left to right
    assert R.replace(b"abcabc", b"bc", b"") == b"aa"     # an empty rep deletes
    assert R.replace(b"abc", b"", b"x") == b"abc"        # an empty search changes nothing
    assert R.replace(b"", b"a", b"x") == b""
    assert R.replace(E3 + b"a" + E3, E3, E4) == E4 + b"a" + E4
    assert R.replace(b"abc", b"abcd", b"x") == b"abc"
    assert R.replace(None, b"a", b"b") is None and R.replace(b"a", None, b"b") is None and R.replace(b"a", b"a", None) is None


def test_translate_rules():
    assert R.translate(b"abcabc", b"ab", b"xy") == b"xycxyc"
    assert R.translate(b"abcd", b"abc", b"x") == b"xd"                       # b, c have no partner: deleted
    assert R.translate(b"aab", b"aa", b"xy") == b"xxb"                       # the first occurrence wins
    assert R.translate(b"abc", b"aab", b"xyz") == b"xzc"                     # ... and the duplicate uses up position 1
    assert R.translate(b"a" + E2 + b"b", b"a" + E2, E4 + b"e") == E4 + b"eb"   # byte lengths change both ways
    assert R.translate(E3 * 2, E3, b"") == b""
    assert R.translate(b"abc", b"", b"xyz") == b"abc"
    assert R.translate(None, b"a", b"b") is None and R.translate(b"a", b"a", None) is None


def test_reverse_ascii_bit_length():
    assert R.reverse(b"abc") == b"cba"
    assert R.reverse(b"a" + E2 + E3 + E4) == E4 + E3 + E2 + b"a"
    assert R.reverse(b"") == b"" and R.reverse(None) is None
    assert R.ascii_(b"") == 0 and R.ascii_(b"A") == 65 and R.ascii_(b"abc") == 97
    assert [R.ascii_(c.encode()) for c in ("\u0080", "߿", "ࠀ", "￿", "\U00010000", "\U0010ffff")] == \
        [0x80, 0x7FF, 0x800, 0xFFFF, 0x10000, 0x10FFFF]
    assert R.ascii_(None) is None
    assert R.bit_length(b"") == 0 and R.bit_length(E4) == 32 and R.bit_length(None) is None


def test_find_in_set_rules():
    assert R.find_in_set(b"ab", b"abc,b,ab,c,def") == 3
    assert R.find_in_set(b"x", b"a,b") == 0
    assert R.find_in_set(b"a,b", b"a,b") == 0      # s holds a comma
    assert R.find_in_set(b"", b"") == 1
    assert R.find_in_set(b"", b"a,,b") == 2        # an empty piece
    assert R.find_in_set(b"", b"a,b,") == 3
    assert R.find_in_set(b"", b"a,b") == 0
    assert R.find_in_set(E3, b"a," + E3) == 2
    assert R.find_in_set(None, b"a") is None and R.find_in_set(b"a", None) is None


def test_trim_with_a_set():
    assert R.trim(b"00120300", b"0") == b"1203"
    assert R.trim(b"00120300", b"0", "left") == b"120300"
    assert R.trim(b"00120300", b"0", "right") == b"001203"
    assert R.trim(b"xyabcyx", b"yx") == b"abc"
    assert R.trim(b"  a  ", b"") == b"  a  "       # an empty set changes nothing
    assert R.trim(b"0000", b"0") == b""
    assert R.trim(E3 + b"a" + E4 + E3, E3 + E4) == b"a"
    assert R.trim(None, b"x") is None and R.trim(b"x", None) is None


# ------------------------------------------------------------------------------------------------------------ planning
SCHEMA = pa.schema([("s", pa.string()), ("t", pa.string()), ("b", pa.binary()), ("i", pa.int64()), ("n", pa.int32()),
                    ("h", pa.int16()), ("f", pa.float64())])
U, I32 = pa.string(), pa.int32()


def _fn(name, *args, t=U):
    return P.scalar_fn(name, list(args), t)


def _lit(v, t=U):
    return P.lit(v, t)


def _i64(e):
    return P.cast(e, pa.int64())


def _explain(plan):
    return runtime.explain(P.task_definition(plan))


def _project(exprs, types=None, src=None):
    src = src or P.ffi_reader(SCHEMA, "t")
    return P.projection(src, exprs, [f"c{i}" for i in range(len(exprs))], types or [U] * len(exprs))


def _lpad(*a):
    return _fn("Lpad", *a)


STRING_FNS = {
    "lpad": _lpad(P.col("s"), _i64(P.col("n")), _lit("0")),
    "lpad_int16_length": _lpad(P.col("s"), P.col("h"), P.col("t")),
    "rpad": _fn("Rpad", P.col("s"), P.col("i"), _lit("xy")),
    "rpad_null_pad": _fn("Rpad", P.col("s"), P.col("i"), _lit(None)),
    "replace": _fn("Replace", P.col("s"), _lit("a"), P.col("t")),
    "replace_of_upper": _fn("Replace", _fn("Upper", P.col("s")), _lit("A"), _lit("x")),
    "translate": _fn("Translate", P.col("s"), _lit("abc"), _lit("xy")),
    "reverse": _fn("Reverse", P.col("s")),
    "reverse_of_substr": _fn("Reverse", P.scalar_fn("Substr", [P.col("s"), _lit(2, pa.int64()), _lit(3, pa.int64())], U)),
    "initcap": _fn("Spark_InitCap", P.col("s")),
    "initcap_of_case": _fn("Spark_InitCap", P.case([(P.is_null(P.col("s")), _lit("none"))], P.col("s"))),
    "lpad_of_lower_trim_coalesce": _lpad(_fn("Lower", _fn("Trim", P.col("s"))), _lit(9, pa.int64()),
                                         P.scalar_fn("Coalesce", [P.col("t"), _lit("-")], U)),
}
NUMBER_FNS = {
    "ascii": _fn("Ascii", P.col("s"), t=I32),
    "bit_length": _fn("BitLength", P.col("s"), t=I32),
    "bit_length_binary": _fn("BitLength", P.col("b"), t=I32),
    "find_in_set": _fn("FindInSet", P.col("s"), _lit("a,b,c"), t=I32),
}
TRIMS = {f"{name}_set": _fn(name, P.col("s"), P.col("t")) for name in ("Trim", "Btrim", "Ltrim", "Rtrim")}


@pytest.mark.parametrize("shape", sorted(STRING_FNS))
def test_string_function_plans_as_a_projection(shape):
    plan = _explain(_project([STRING_FNS[shape], P.col("i")], [U, pa.int64()]))["plan"]
    assert plan["op"] == "ProjectExec"
    assert plan["schema"][0][1] == "utf8", plan["schema"]


@pytest.mark.parametrize("shape", sorted(STRING_FNS))
def test_string_function_plans_as_a_piece_and_a_digest_argument(shape):
    e = STRING_FNS[shape]
    exprs = [_fn("Spark_StringConcat", _lit("<"), e, P.col("s")), _fn("Spark_StringConcatWs", _lit("|"), P.col("s"), e, _lit(None)),
             _fn("Spark_MD5", e), _fn("Spark_Sha256", P.try_cast(e, U)), P.try_cast(e, U)]
    plan = _explain(_project(exprs))["plan"]
    assert [c[1] for c in plan["schema"]] == ["utf8"] * len(exprs)


@pytest.mark.parametrize("shape", sorted(NUMBER_FNS) + sorted(TRIMS))
def test_number_functions_and_trim_plan_anywhere(shape):
    e = {**NUMBER_FNS, **TRIMS}[shape]
    rt = U if shape in TRIMS else I32
    plan = _explain(_project([e], [rt]))["plan"]
    assert plan["schema"][0][1] == ("utf8" if shape in TRIMS else "int32"), plan["schema"]
    src = P.ffi_reader(SCHEMA, "t")
    probe = _lit("x") if shape in TRIMS else _lit(3, I32)
    _explain(P.filter_(src, [P.binary("Eq", e, probe)]))
    _explain(_project([P.case([(P.binary("Gt", P.col("i"), _lit(0, pa.int64())), e)], probe)], [rt]))
    _explain(P.agg(src, [e], ["k"], [P.agg_expr("COUNT", [P.col("i")], pa.int64())], ["c"], ["PARTIAL"]))


def test_every_string_function_in_one_projection_and_as_keys():
    _explain(_project(list(STRING_FNS.values())))
    src = P.ffi_reader(SCHEMA, "t")
    key = _lpad(P.col("s"), _lit(12, pa.int64()), _lit("*"))
    _explain(P.agg(src, [key, _fn("Spark_InitCap", P.col("t"))], ["k", "j"], [P.agg_expr("COUNT", [P.col("i")], pa.int64())], ["c"], ["PARTIAL"]))
    _explain(P.shuffle_writer(src, P.hash_repartition([_fn("Replace", P.col("s"), _lit("a"), _lit("b"))], 4), "/tmp/x.data", "/tmp/x.index"))
    _explain(P.sort(src, [P.sort_expr(_fn("Reverse", P.col("s")))]))


REJECTED = {
    "lpad_in_comparison": ("Lpad", P.binary("Eq", _lpad(P.col("s"), P.col("i"), _lit("0")), _lit("x"))),
    "replace_in_case": ("Replace", P.case([(P.is_null(P.col("s")), _fn("Replace", P.col("s"), _lit("a"), _lit("b")))], P.col("s"))),
    "upper_of_lpad": ("Lpad", _fn("Upper", _lpad(P.col("s"), P.col("i"), _lit("0")))),
    "lpad_of_replace": ("Replace", _lpad(_fn("Replace", P.col("s"), _lit("a"), _lit("b")), P.col("i"), _lit("0"))),
    "reverse_of_initcap": ("Spark_InitCap", _fn("Reverse", _fn("Spark_InitCap", P.col("s")))),
    "translate_of_concat": ("Spark_StringConcat", _fn("Translate", _fn("Spark_StringConcat", P.col("s")), _lit("a"), _lit("b"))),
    "repeat_of_reverse": ("Reverse", _fn("Spark_StringRepeat", _fn("Reverse", P.col("s")), _lit(2, I32))),
    "substr_of_rpad": ("Rpad", P.scalar_fn("Substr", [_fn("Rpad", P.col("s"), P.col("i"), _lit("0")), _lit(1, pa.int64())], U)),
    "ascii_of_lpad": ("Lpad", _fn("Ascii", _lpad(P.col("s"), P.col("i"), _lit("0")), t=I32)),
    "trim_set_of_reverse": ("Reverse", _fn("Trim", P.col("s"), _fn("Reverse", P.col("t")))),
    "lpad_float_length": ("Lpad", _lpad(P.col("s"), P.col("f"), _lit("0"))),
    "lpad_binary": ("Lpad", _lpad(P.col("b"), P.col("i"), _lit("0"))),
    "replace_int_search": ("Replace", _fn("Replace", P.col("s"), P.col("i"), _lit("0"))),
    "reverse_two_arguments": ("Reverse", _fn("Reverse", P.col("s"), P.col("t"))),
    "ascii_binary": ("Ascii", _fn("Ascii", P.col("b"), t=I32)),
    "find_in_set_int": ("FindInSet", _fn("FindInSet", P.col("s"), P.col("n"), t=I32)),
    "bit_length_int": ("BitLength", _fn("BitLength", P.col("i"), t=I32)),
    "trim_int_set": ("Trim", _fn("Trim", P.col("s"), P.col("n"))),
}


@pytest.mark.parametrize("shape", sorted(REJECTED))
def test_rejected_positions_name_the_function(shape):
    name, expr = REJECTED[shape]
    with pytest.raises(runtime.AuronError, match=name):
        _explain(_project([expr]))


@pytest.mark.parametrize("name", ["Lpad", "Rpad", "Replace", "Translate", "Reverse", "Spark_InitCap"])
def test_string_function_in_a_filter_is_rejected(name):
    args = {"Lpad": [P.col("s"), P.col("i"), _lit("0")], "Rpad": [P.col("s"), P.col("i"), _lit("0")],
            "Replace": [P.col("s"), _lit("a"), _lit("b")], "Translate": [P.col("s"), _lit("a"), _lit("b")]}.get(name, [P.col("s")])
    src = P.ffi_reader(SCHEMA, "t")
    with pytest.raises(runtime.AuronError, match=name):
        _explain(P.filter_(src, [P.binary("Eq", _fn(name, *args), _lit("x"))]))
