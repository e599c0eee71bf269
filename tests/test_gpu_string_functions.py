"""lpad, rpad, replace, translate, reverse, initcap, ascii, bit_length, find_in_set and trim with a character set on the GPU,
value by value against the plain-Python reference in string_reference.py (its docstring states the semantics), in every position
the planner accepts them: a whole projection expression, a piece of concat / concat_ws, a digest's argument, and for the
functions that return a number or a view also a Filter, CASE and comparisons."""
import hashlib

import numpy as np
import pyarrow as pa
import pytest

import oracle
import string_reference as R
from auron_b200 import proto as P
from auron_b200 import runtime
from helpers import assert_same_rows, run
from test_gpu_shuffle import read_shuffle_files

pytestmark = pytest.mark.gpu

U, I32, I64 = pa.string(), pa.int32(), pa.int64()


def fn(name, *args, t=U):
    return P.scalar_fn(name, list(args), t)


def lit(v, t=U):
    return P.lit(v, t)


def project(t, exprs, types, src=None):
    src = src or P.ffi_reader(t.schema, "t")
    return P.projection(src, exprs, [f"c{i}" for i in range(len(exprs))], types)


def as_bytes(col):   # utf8 results compared as their bytes, so that a malformed value cannot hide behind a decode
    return col.cast(pa.binary()).to_pylist() if pa.types.is_string(col.type) else col.to_pylist()


def enc(v):
    return None if v is None else v.encode()


def md5(v):
    return None if v is None else hashlib.md5(v).hexdigest().encode()


def concat(*vals):
    return None if any(v is None for v in vals) else b"".join(vals)


def concat_ws(sep, *vals):
    return sep.join(v for v in vals if v is not None)


# ---------------------------------------------------------------------------------------------- reference goldens
def test_initcap_goldens():
    # spark_initcap.rs:80-118
    inp = [None, "", "hI THOmAS", "James-Smith", "michael rose", "a1b2   c3D4", " ---abc--- ABC --ABC-- a-b A B eB Ac c d", " 世  界  世界 ",
           "abC c3D4"]
    exp = [None, "", "Hi Thomas", "James-smith", "Michael Rose", "A1b2   C3d4", " ---abc--- Abc --abc-- A-b A B Eb Ac C D", " 世  界  世界 ",
           "Abc C3d4"]
    t = pa.table({"s": pa.array(inp)})
    out = run(project(t, [fn("Spark_InitCap", P.col("s"))], [U]), {"t": t})
    assert out.column(0).to_pylist() == exp
    assert out.schema.field(0).type == U


def test_hand_computed_values():
    t = pa.table({"s": pa.array(["abc", "aaa", "00120300", "", "a,b", None]), "n": pa.array([5, 2, 3, 0, -1, 4], type=I64)})
    exprs = [fn("Lpad", P.col("s"), P.col("n"), lit("xy")), fn("Rpad", P.col("s"), P.col("n"), lit("")),
             fn("Replace", P.col("s"), lit("aa"), lit("b")), fn("Translate", P.col("s"), lit("a0"), lit("Z")),
             fn("Reverse", P.col("s")), fn("Trim", P.col("s"), lit("0")), fn("Ltrim", P.col("s"), lit("0")), fn("Rtrim", P.col("s"), lit("0")),
             fn("Ascii", P.col("s"), t=I32), fn("BitLength", P.col("s"), t=I32), fn("FindInSet", lit("b"), P.col("s"), t=I32),
             fn("FindInSet", lit(""), P.col("s"), t=I32)]
    out = run(project(t, exprs, [U] * 8 + [I32] * 4), {"t": t})
    assert out.column(0).to_pylist() == ["xyabc", "aa", "001", "", "", None]
    assert out.column(1).to_pylist() == ["abc", "aa", "001", "", "", None]
    assert out.column(2).to_pylist() == ["abc", "ba", "00120300", "", "a,b", None]
    assert out.column(3).to_pylist() == ["Zbc", "ZZZ", "123", "", "Z,b", None]   # '0' has no partner in 'Z': deleted
    assert out.column(4).to_pylist() == ["cba", "aaa", "00302100", "", "b,a", None]
    assert out.column(5).to_pylist() == ["abc", "aaa", "1203", "", "a,b", None]
    assert out.column(6).to_pylist() == ["abc", "aaa", "120300", "", "a,b", None]
    assert out.column(7).to_pylist() == ["abc", "aaa", "001203", "", "a,b", None]
    assert out.column(8).to_pylist() == [97, 97, 48, 0, 97, None]
    assert out.column(9).to_pylist() == [24, 24, 64, 0, 24, None]
    assert out.column(10).to_pylist() == [0, 0, 0, 0, 2, None]
    assert out.column(11).to_pylist() == [0, 0, 0, 1, 0, None]
    assert [f.type for f in out.schema] == [U] * 8 + [I32] * 4


# ---------------------------------------------------------------------------------------------- fuzz
WIDE = ["\u0080", "߿", "ࠀ", "￿", "\U00010000", "\U0010ffff"]   # the first and last code point of each UTF-8 length
ALPHABET = list("abcABCxyz 0,é天😁") + WIDE
SHORT = list("ab,0 é") + ["\U0010ffff", "ࠀ"]


def _strings(rng, n, alphabet, max_chars, p_null=0.05):
    lens = rng.integers(0, max_chars + 1, n)
    pool = rng.choice(np.array(alphabet, dtype=object), int(lens.sum()))
    ends = np.cumsum(lens)
    vals = ["".join(pool[e - k:e]) for e, k in zip(ends, lens)]
    return pa.array(vals, type=U, mask=rng.random(n) < p_null)


def _fuzz_table(n, seed):
    rng = np.random.default_rng(seed)
    return pa.table({"s": _strings(rng, n, ALPHABET, 40), "t": _strings(rng, n, SHORT, 3), "u": _strings(rng, n, ALPHABET, 4),
                     "n": pa.array(rng.integers(-3, 50, n), type=I32, mask=rng.random(n) < 0.05),
                     "k": pa.array(rng.integers(0, 100, n), type=I32)})


def _fuzz_cases():
    """(expression, output type, reference of one row {s, t, u, n})"""
    s, t, u, n = P.col("s"), P.col("t"), P.col("u"), P.col("n")
    n64 = P.cast(n, I64)
    lpad = fn("Lpad", s, n64, t)
    return [
        (lpad, U, lambda r: R.lpad(r["s"], r["n"], r["t"])),
        (fn("Rpad", s, n, u), U, lambda r: R.rpad(r["s"], r["n"], r["u"])),
        (fn("Lpad", t, n64, s), U, lambda r: R.lpad(r["t"], r["n"], r["s"])),
        (fn("Lpad", s, lit(12, I64), lit("0")), U, lambda r: R.lpad(r["s"], 12, b"0")),
        (fn("Replace", s, t, u), U, lambda r: R.replace(r["s"], r["t"], r["u"])),
        (fn("Replace", s, lit("a"), lit("\U0010ffff")), U, lambda r: R.replace(r["s"], b"a", enc("\U0010ffff"))),
        (fn("Translate", s, t, u), U, lambda r: R.translate(r["s"], r["t"], r["u"])),
        (fn("Translate", s, u, t), U, lambda r: R.translate(r["s"], r["u"], r["t"])),
        (fn("Reverse", s), U, lambda r: R.reverse(r["s"])),
        (fn("Spark_InitCap", s), U, lambda r: R.initcap(r["s"])),
        (fn("Ascii", s, t=I32), I32, lambda r: R.ascii_(r["s"])),
        (fn("BitLength", s, t=I32), I32, lambda r: R.bit_length(r["s"])),
        (fn("FindInSet", t, s, t=I32), I32, lambda r: R.find_in_set(r["t"], r["s"])),
        (fn("Trim", s, t), U, lambda r: R.trim(r["s"], r["t"])),
        (fn("Btrim", s, u), U, lambda r: R.trim(r["s"], r["u"])),
        (fn("Ltrim", s, t), U, lambda r: R.trim(r["s"], r["t"], "left")),
        (fn("Rtrim", s, t), U, lambda r: R.trim(r["s"], r["t"], "right")),
        # the case marks of upper / lower are read, not only copied
        (fn("Replace", fn("Upper", s), lit("A"), lit("x")), U, lambda r: R.replace(R.upper(r["s"]), b"A", b"x")),
        (fn("Lpad", fn("Lower", s), n64, fn("Upper", t)), U, lambda r: R.lpad(R.lower(r["s"]), r["n"], R.upper(r["t"]))),
        (fn("Translate", fn("Lower", s), lit("abc"), fn("Upper", u)), U, lambda r: R.translate(R.lower(r["s"]), b"abc", R.upper(r["u"]))),
        (fn("FindInSet", fn("Upper", t), fn("Upper", s), t=I32), I32, lambda r: R.find_in_set(R.upper(r["t"]), R.upper(r["s"]))),
        (fn("Trim", fn("Lower", s), lit("ab")), U, lambda r: R.trim(R.lower(r["s"]), b"ab")),
        # pieces: concat propagates NULL, concat_ws skips it with its separator
        (fn("Spark_StringConcat", lpad, lit("|"), fn("Reverse", s)), U,
         lambda r: concat(R.lpad(r["s"], r["n"], r["t"]), b"|", R.reverse(r["s"]))),
        (fn("Spark_StringConcatWs", lit("||"), fn("Translate", s, t, u), fn("Spark_InitCap", u), fn("Rpad", s, n, u), t), U,
         lambda r: concat_ws(b"||", R.translate(r["s"], r["t"], r["u"]), R.initcap(r["u"]), R.rpad(r["s"], r["n"], r["u"]), r["t"])),
        (fn("Spark_MD5", lpad), U, lambda r: md5(R.lpad(r["s"], r["n"], r["t"]))),
        (fn("Spark_Sha256", fn("Spark_StringConcatWs", lit("-"), fn("Replace", s, t, u), s)), U,
         lambda r: hashlib.sha256(concat_ws(b"-", R.replace(r["s"], r["t"], r["u"]), r["s"])).hexdigest().encode()),
    ]


def _rows(t):
    cols = {k: as_bytes(t.column(k)) for k in ("s", "t", "u")}
    cols["n"] = t.column("n").to_pylist()
    return [dict(zip(cols, v)) for v in zip(*cols.values())]


def _check(got, t, cases):
    rows = _rows(t)
    assert got.num_rows == len(rows)
    for k, (_, typ, ref) in enumerate(cases):
        assert got.schema.field(k).type == typ, k
        exp = [ref(r) for r in rows]
        g = as_bytes(got.column(k))
        bad = [i for i, (a, b) in enumerate(zip(g, exp)) if a != b]
        assert not bad, (k, len(bad), [(rows[i], g[i], exp[i]) for i in bad[:3]])


def test_fuzz_several_batches():
    t = _fuzz_table(200_000, seed=41)
    cases = _fuzz_cases()
    got = run(project(t, [c[0] for c in cases], [c[1] for c in cases]), {"t": t}, chunk=70_000)
    _check(got, t, cases)


def test_fuzz_below_a_filter():
    t = _fuzz_table(60_000, seed=42)
    cases = _fuzz_cases()
    flt = P.filter_(P.ffi_reader(t.schema, "t"), [P.binary("Lt", P.col("k"), lit(37, I32))])   # the selection path
    got = run(project(t, [c[0] for c in cases], [c[1] for c in cases], src=flt), {"t": t}, chunk=25_000)
    _check(got, t.filter(pa.array(np.asarray(t.column("k")) < 37)), cases)


def test_numbers_and_trim_in_a_filter_and_in_case():
    t = _fuzz_table(50_000, seed=43)
    rows = _rows(t)
    s, tt = P.col("s"), P.col("t")
    src = P.ffi_reader(t.schema, "t")
    preds = [([P.binary("GtEq", fn("Ascii", s, t=I32), lit(128, I32))], lambda r: (R.ascii_(r["s"]) or 0) >= 128),
             ([P.binary("Gt", fn("FindInSet", tt, s, t=I32), lit(1, I32))], lambda r: (R.find_in_set(r["t"], r["s"]) or 0) > 1),
             ([P.binary("Eq", fn("Trim", s, tt), s)], lambda r: r["s"] is not None and r["t"] is not None and R.trim(r["s"], r["t"]) == r["s"]),
             ([P.binary("Lt", fn("BitLength", s, t=I32), lit(80, I32)), P.binary("NotEq", fn("Rtrim", s, lit("0 ")), lit(""))],
              lambda r: r["s"] is not None and 8 * len(r["s"]) < 80 and R.trim(r["s"], b"0 ", "right") != b"")]
    for k, (pred, ref) in enumerate(preds):
        got = run(project(t, [s], [U], src=P.filter_(src, pred)), {"t": t}, chunk=20_000)
        exp = [r["s"] for r in rows if ref(r)]
        assert as_bytes(got.column(0)) == exp, k
        assert 0 < len(exp) < len(rows), k
    gt = lambda a, b: P.binary("Gt", a, b)   # noqa: E731
    case_n = P.case([(gt(fn("Ascii", s, t=I32), lit(127, I32)), lit(1, I32)), (gt(fn("FindInSet", tt, s, t=I32), lit(0, I32)), lit(2, I32))],
                    lit(0, I32))
    case_s = P.case([(gt(fn("BitLength", s, t=I32), lit(100, I32)), fn("Ltrim", s, tt))], fn("Rtrim", s, lit("abc")))
    got = run(project(t, [case_n, case_s], [I32, U]), {"t": t}, chunk=20_000)
    exp_n = [1 if (R.ascii_(r["s"]) or 0) > 127 else 2 if (R.find_in_set(r["t"], r["s"]) or 0) > 0 else 0 for r in rows]
    exp_s = [R.trim(r["s"], r["t"], "left") if r["s"] is not None and 8 * len(r["s"]) > 100 else R.trim(r["s"], b"abc", "right") for r in rows]
    assert got.column(0).to_pylist() == exp_n
    assert as_bytes(got.column(1)) == exp_s


# ---------------------------------------------------------------------------------------------- query level
def test_group_by_lpad_partial_and_final():
    rng = np.random.default_rng(51)
    n = 120_000
    words = ["1", "22", "é", "天地", "", "abcdefghijk", "\U0010ffff"]
    t = pa.table({"s": pa.array([words[int(k)] for k in rng.integers(0, len(words), n)], mask=rng.random(n) < 0.02),
                  "w": pa.array(rng.integers(4, 7, n), type=I32), "v": pa.array(rng.integers(0, 10, n), type=I64)})
    key = fn("Lpad", P.col("s"), P.col("w"), lit("0é"))
    partial = P.agg(P.ffi_reader(t.schema, "t"), [key], ["k"], [P.agg_expr("COUNT", [P.col("v")], I64)], ["c"], ["PARTIAL"])
    final = P.agg(partial, [P.col("k")], ["k"], [P.agg_expr("COUNT", [P.lit(None, pa.null())], I64)], ["c"], ["FINAL"])
    got = run(final, {"t": t}, chunk=40_000)
    counts = {}
    for s, w in zip(as_bytes(t.column("s")), t.column("w").to_pylist()):
        k = R.lpad(s, w, enc("0é"))
        counts[k] = counts.get(k, 0) + 1
    exp = pa.table({"k": pa.array([None if k is None else k.decode() for k in counts], type=U), "c": pa.array(list(counts.values()), type=I64)})
    assert_same_rows(got, exp)


def test_hash_shuffle_partitioned_on_replace(tmp_path):
    rng = np.random.default_rng(52)
    n, nparts = 80_000, 16
    t = pa.table({"a": pa.array([f"a{int(k)}-é" for k in rng.integers(0, 3000, n)], mask=rng.random(n) < 0.03),
                  "x": pa.array(np.arange(n), type=I64)})
    data, index = str(tmp_path / "r.data"), str(tmp_path / "r.index")
    key = fn("Replace", P.col("a"), lit("1"), lit("ࠀ"))
    run(P.shuffle_writer(P.ffi_reader(t.schema, "t"), P.hash_repartition([key], nparts), data, index), {"t": t}, chunk=30_000)
    parts, _ = read_shuffle_files(data, index, t.schema)
    keys = pa.array([None if v is None else v.replace("1", "ࠀ") for v in t.column("a").to_pylist()], type=U)
    pid = oracle.partition_ids([keys], nparts)
    for p in range(nparts):
        assert_same_rows(parts[p], t.filter(pa.array(pid == p)))
    assert sum(x.num_rows for x in parts) == n


def test_padding_past_2_gib_fails_the_batch():
    t = pa.table({"s": pa.array(["abc"])})
    for n in (2**31, 2**63 - 1):
        for name in ("Lpad", "Rpad"):
            with pytest.raises(runtime.AuronError, match="utf8 column exceeds 2 GiB in one batch"):
                run(project(t, [fn(name, P.col("s"), lit(n, I64), lit("x"))], [U]), {"t": t})
    # the same plan with a length that fits runs
    out = run(project(t, [fn("Lpad", P.col("s"), lit(1000, I64), lit("xy"))], [U]), {"t": t})
    assert out.column(0).to_pylist() == [R.lpad(b"abc", 1000, b"xy").decode()]
