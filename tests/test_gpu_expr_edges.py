"""The expression VM (k_expr.cu) against the plain-Python reference of tests/expr_reference.py, at the edges of every type.

Each case packs many expressions into one projection over the cross product of the operand type's edge values plus seeded random
fill and NULLs, and compares every value exactly: integers, decimals (as unscaled ints), floats by their bits (any NaN matches
any NaN; the sign of zero counts), strings by their bytes.  Each case runs
  * with and without a Filter below the projection, so the selection path of the VM runs too,
  * in both kernel instantiations: an extra decimal output column sends a program through vm_kernel<true>.
Decimal + - * are built in the reference's plan shape Cast(BinaryExpr(Cast(lhs, rt), rhs), rt) (NativeConverters.scala)."""
import decimal
import os
import random

import numpy as np
import pyarrow as pa
import pytest

import expr_reference as R
from auron_b200 import proto as P
from auron_b200 import runtime
from helpers import run
from key_reference import INT_BITS, edge_values, unscaled_to_decimal

pytestmark = pytest.mark.gpu

_INT_PA = {"int8": pa.int8(), "int16": pa.int16(), "int32": pa.int32(), "int64": pa.int64()}
_FLOAT_PA = {"float32": pa.float32(), "float64": pa.float64()}
_KEEP = 3                                              # the Filter below a case keeps rows whose id is not a multiple of 3


# -------------------------------------------------------------------------------------------- arrow <-> canonical values
def _arrow(vals, t):
    """canonical values -> an Arrow array of type t (str for ints / floats, ("dec", p, s) for decimals, or a pa type)"""
    if t in _INT_PA:
        return pa.array(vals, type=_INT_PA[t])
    if t in _FLOAT_PA:
        dt = np.uint32 if t == "float32" else np.uint64
        bits = np.array([0 if v is None else v for v in vals], dtype=dt)
        return pa.array(bits.view(np.float32 if t == "float32" else np.float64), mask=np.array([v is None for v in vals]))
    if isinstance(t, tuple):
        return pa.array([None if v is None else unscaled_to_decimal(v, t[2]) for v in vals], type=pa.decimal128(t[1], t[2]))
    return pa.array(vals, type=t)


def _canon(col: pa.ChunkedArray, t):
    """an output column -> canonical values"""
    a = col.combine_chunks()
    if t in _FLOAT_PA:
        bits = np.asarray(a.fill_null(0).to_numpy(zero_copy_only=False)).view(np.uint32 if t == "float32" else np.uint64)
        return [int(b) if ok else None for b, ok in zip(bits, a.is_valid().to_pylist())]
    if isinstance(t, tuple):
        with decimal.localcontext() as ctx:
            ctx.prec = 80
            return [None if v is None else int(v.scaleb(t[2])) for v in a.to_pylist()]
    if pa.types.is_string(a.type):
        return [None if v is None else v.encode() for v in a.to_pylist()]
    return a.to_pylist()


def _is_nan(b, t) -> bool:
    mant, exp_mask = (23, 0xFF) if t == "float32" else (52, 0x7FF)
    return b is not None and (b >> mant) & exp_mask == exp_mask and b & ((1 << mant) - 1) != 0


def _same(got, exp, t):
    if t in _FLOAT_PA:
        return got == exp or (_is_nan(got, t) and _is_nan(exp, t))   # NaN payloads are not pinned
    return got == exp


def _pa_type(t):
    if t in _INT_PA:
        return _INT_PA[t]
    if t in _FLOAT_PA:
        return _FLOAT_PA[t]
    if isinstance(t, tuple):
        return pa.decimal128(t[1], t[2])
    return t


def _column(t, n, seed, null_rate=0.05):
    """edge values first (so that pairs of columns built with different seeds cross them), then random fill and NULLs"""
    rng = random.Random(seed)
    edges = edge_values(t) if not isinstance(t, tuple) else _dec_edges(t[1])
    out = []
    for i in range(n):
        u = rng.random()
        if u < null_rate:
            out.append(None)
        elif u < 0.5:
            out.append(rng.choice(edges))
        elif t in INT_BITS:
            b = INT_BITS[t]
            out.append(rng.randrange(-(1 << (b - 1)), 1 << (b - 1)) if rng.random() < 0.5 else rng.randrange(-70, 70))
        elif t in _FLOAT_PA:
            x = rng.choice([rng.uniform(-1e6, 1e6), rng.uniform(-2, 2), rng.uniform(-1e300, 1e300), rng.uniform(-1e-300, 1e-300)])
            out.append(R.from_float(x, t))
        else:
            m = 10 ** t[1] - 1
            out.append(rng.randrange(-m, m + 1) if rng.random() < 0.5 else rng.randrange(-10**6, 10**6))
    return out


def _dec_edges(p):
    m = 10 ** p - 1
    return [m, -m, 1, -1, 0, m // 2, -(m // 2), 10 ** (p - 1), -(10 ** (p - 1))]


def _cross(t, u=None):
    """every (edge, edge) pair of types t and u"""
    ea = edge_values(t) + [None]
    eb = edge_values(u or t) + [None]
    return [a for a in ea for _ in eb], [b for _ in ea for b in eb]


def _project(table, exprs, types, filtered, hi, chunk=None):
    """run Project[exprs] (optionally over Filter[id % 3 != 0]); `hi` adds a decimal output so the program runs vm_kernel<true>.
    Returns the output columns as canonical values and the row ids that reached the projection."""
    src = P.ffi_reader(table.schema, "t")
    if filtered:
        src = P.filter_(src, [P.binary("NotEq", P.binary("Modulo", P.col("id"), P.lit(_KEEP, pa.int64())), P.lit(0, pa.int64()))])
    exprs = list(exprs) + [P.col("id")] + ([P.try_cast(P.col("id"), pa.decimal128(20, 0))] if hi else [])
    names = [f"o{k}" for k in range(len(exprs))]
    ptypes = [_pa_type(t) for t in types] + [pa.int64()] + ([pa.decimal128(20, 0)] if hi else [])
    out = run(P.projection(src, exprs, names, ptypes), {"t": table}, chunk=chunk)
    ids = out[names[len(types)]].to_pylist()
    if hi:
        assert _canon(out[names[-1]], ("dec", 20, 0)) == ids
    exp_ids = [i for i in range(table.num_rows) if not filtered or i % _KEEP != 0]
    assert ids == exp_ids
    return [_canon(out[names[k]], t) for k, t in enumerate(types)], ids


def _check(got_cols, exp_fns, rows, ids, types, labels):
    for g, f, t, label in zip(got_cols, exp_fns, types, labels):
        for pos, i in enumerate(ids):
            e = f(*rows[i])
            if not _same(g[pos], e, t):
                raise AssertionError(f"{label}: row {i} inputs {rows[i]} -> got {g[pos]}, expected {e}")


MODES = [pytest.param(f, h, id=f"{'filter' if f else 'plain'}-{'hi' if h else 'lo'}") for f in (False, True) for h in (False, True)]
BIN_INT = ["Plus", "Minus", "Multiply", "Divide", "Modulo", "BitwiseAnd", "BitwiseOr", "BitwiseXor", "BitwiseShiftLeft", "BitwiseShiftRight"]
CMPS = ["Eq", "NotEq", "Lt", "LtEq", "Gt", "GtEq", "IsNotDistinctFrom"]


# -------------------------------------------------------------------------------------------- integers
@pytest.mark.parametrize("filtered,hi", MODES)
@pytest.mark.parametrize("t", list(INT_BITS))
def test_integer_ops_at_the_edges(t, filtered, hi):
    xa, xb = _cross(t)
    xb = [b if i % 5 else (None if b is None else b % 70) for i, b in enumerate(xb)]   # shift counts past the width and back
    n = 3000
    a = xa + _column(t, n, 1)
    b = xb + _column(t, n, 2)
    table = pa.table({"a": _arrow(a, t), "b": _arrow(b, t), "id": pa.array(range(len(a)), type=pa.int64())})
    A, B = P.col("a"), P.col("b")
    exprs, types, fns, labels = [], [], [], []
    for op in BIN_INT:
        rhs = P.scalar_fn("Spark_NullIfZero", [B], _INT_PA[t]) if op in ("Divide", "Modulo") else B
        exprs.append(P.binary(op, A, rhs))
        types.append(t)
        fns.append(lambda x, y, op=op: R.arith(op, x, y, t))
        labels.append(op)
    for op in CMPS:
        exprs.append(P.binary(op, A, B))
        types.append(pa.bool_())
        fns.append(lambda x, y, op=op: R.compare(op, x, y, t))
        labels.append(op)
    exprs += [P.negative(A), P.scalar_fn("Abs", [A], _INT_PA[t]), P.scalar_fn("NullIf", [A, B], _INT_PA[t]),
              P.scalar_fn("Coalesce", [A, B], _INT_PA[t])]
    types += [t] * 4
    fns += [lambda x, y: R.negate(x, t), lambda x, y: None if x is None else R.wrap(abs(x), INT_BITS[t]),
            lambda x, y: R.null_if(x, y), lambda x, y: R.coalesce(x, y)]
    labels += ["Negative", "Abs", "NullIf", "Coalesce"]
    got, ids = _project(table, exprs, types, filtered, hi)
    _check(got, fns, list(zip(a, b)), ids, types, labels)


def test_integer_ops_turn_the_grid_stride_loop():
    # more rows than sm_count x 6 blocks x 256 threads (203k on 132 SMs): the kernel's grid-stride loop runs a second round
    n = 250_000
    a, b = _column("int32", n, 11), _column("int32", n, 12)
    table = pa.table({"a": _arrow(a, "int32"), "b": _arrow(b, "int32"), "id": pa.array(range(n), type=pa.int64())})
    A, B = P.col("a"), P.col("b")
    ops = ["Plus", "Minus", "Multiply", "BitwiseXor", "BitwiseShiftLeft"]
    for filtered in (False, True):
        got, ids = _project(table, [P.binary(op, A, B) for op in ops], ["int32"] * len(ops), filtered, False)
        _check(got, [lambda x, y, op=op: R.arith(op, x, y, "int32") for op in ops], list(zip(a, b)), ids, ["int32"] * len(ops), ops)


@pytest.mark.parametrize("filtered,hi", MODES)
@pytest.mark.parametrize("t", ["int8", "int16"])
def test_narrow_integer_widening_against_int64(t, filtered, hi):
    # int8 / int16 operands against an int64 column are widened before the op: no wrap at the narrow width
    xa, xb = _cross(t, "int64")
    table = pa.table({"a": _arrow(xa, t), "b": _arrow(xb, "int64"), "id": pa.array(range(len(xa)), type=pa.int64())})
    ops = ["Plus", "Minus", "Multiply"]
    got, ids = _project(table, [P.binary(op, P.col("a"), P.col("b")) for op in ops], ["int64"] * 3, filtered, hi)
    _check(got, [lambda x, y, op=op: R.arith(op, x, y, "int64") for op in ops], list(zip(xa, xb)), ids, ["int64"] * 3, ops)


# -------------------------------------------------------------------------------------------- floats
@pytest.mark.parametrize("filtered,hi", MODES)
@pytest.mark.parametrize("t", list(_FLOAT_PA))
def test_float_ops_at_the_edges(t, filtered, hi):
    xa, xb = _cross(t)
    a = xa + _column(t, 2000, 3)
    b = xb + _column(t, 2000, 4)
    table = pa.table({"a": _arrow(a, t), "b": _arrow(b, t), "id": pa.array(range(len(a)), type=pa.int64())})
    A, B = P.col("a"), P.col("b")
    ops = ["Plus", "Minus", "Multiply", "Divide", "Modulo"]
    exprs = [P.binary(op, A, B) for op in ops] + [P.binary(op, A, B) for op in CMPS] + [
        P.negative(A), P.scalar_fn("Spark_NormalizeNanAndZero", [A], _FLOAT_PA[t]), P.scalar_fn("Spark_IsNaN", [A], pa.bool_()),
        P.scalar_fn("Coalesce", [A, B], _FLOAT_PA[t])]
    types = [t] * len(ops) + [pa.bool_()] * len(CMPS) + [t, t, pa.bool_(), t]
    fns = [lambda x, y, op=op: R.arith(op, x, y, t) for op in ops] + [lambda x, y, op=op: R.compare(op, x, y, t) for op in CMPS] + [
        lambda x, y: R.negate(x, t), lambda x, y: R.normalize_nan_and_zero(x, t),
        lambda x, y: x is not None and R.to_float(x, t) != R.to_float(x, t), lambda x, y: R.coalesce(x, y)]
    got, ids = _project(table, exprs, types, filtered, hi)
    _check(got, fns, list(zip(a, b)), ids, types, ops + CMPS + ["Negative", "NormalizeNanAndZero", "IsNaN", "Coalesce"])


# math functions and Power are compared with numpy (glibc) within an ulp bound: the CUDA C Programming Guide's table of double
# precision functions gives sqrt 0 ulp and exp / log / log2 / log10 / sin / cos / tan / asin / acos / atan / pow at most 2 ulp,
# glibc is within 1 ulp, so two correct results are at most 3 ulp apart; sqrt, ceil, floor, trunc and signum are exact
_MATH = {"Sqrt": (np.sqrt, 0), "Exp": (np.exp, 3), "Ln": (np.log, 3), "Log10": (np.log10, 3), "Log2": (np.log2, 3), "Sin": (np.sin, 3),
         "Cos": (np.cos, 3), "Tan": (np.tan, 3), "Asin": (np.arcsin, 3), "Acos": (np.arccos, 3), "Atan": (np.arctan, 3),
         "Ceil": (np.ceil, 0), "Floor": (np.floor, 0), "Trunc": (np.trunc, 0),
         "Signum": (lambda x: np.where(x > 0, 1.0, np.where(x < 0, -1.0, x)), 0)}   # signum keeps -0.0 and NaN


def _ulps(x: float, y: float) -> int:
    if np.isnan(x) and np.isnan(y):
        return 0
    if np.isinf(x) or np.isinf(y) or np.isnan(x) or np.isnan(y):
        return 0 if x == y else 1 << 62
    bx, by = R.total_order(R.from_float(x, "float64"), 64), R.total_order(R.from_float(y, "float64"), 64)
    return abs(bx - by)


@pytest.mark.parametrize("filtered", [False, True])
def test_math_functions_and_power_within_ulps(filtered):
    t = "float64"
    xs = [R.bits_f64(v) for v in edge_values(t)] + [0.5, -0.5, 1e-310, 700.0, -745.0, 1e22, 3.0, 0.1, 2.0 ** 0.5]
    rng = random.Random(5)
    xs += [rng.uniform(-1, 1) for _ in range(400)] + [rng.uniform(-50, 50) for _ in range(400)] + [rng.uniform(0, 1e6) for _ in range(200)]
    ys = [rng.choice([0.5, 2.0, -1.0, 3.0, 0.0, -0.0, 1e-3, rng.uniform(-4, 4)]) for _ in xs]
    table = pa.table({"a": pa.array(xs), "b": pa.array(ys), "id": pa.array(range(len(xs)), type=pa.int64())})
    names = list(_MATH)
    exprs = [P.scalar_fn(f, [P.col("a")], pa.float64()) for f in names] + [P.scalar_fn("Power", [P.col("a"), P.col("b")], pa.float64())]
    got, ids = _project(table, exprs, [t] * len(exprs), filtered, False)
    x = np.array(xs)[ids]
    with np.errstate(all="ignore"):
        for k, f in enumerate(names):
            fn, tol = _MATH[f]
            exp = fn(x)
            for i, (g, e) in enumerate(zip(got[k], exp)):
                assert _ulps(R.bits_f64(g), float(e)) <= tol, (f, x[i], R.bits_f64(g), float(e))
        exp = np.power(x, np.array(ys)[ids])
        for i, (g, e) in enumerate(zip(got[-1], exp)):
            assert _ulps(R.bits_f64(g), float(e)) <= 3, ("Power", x[i], ys[ids[i]], R.bits_f64(g), float(e))


# -------------------------------------------------------------------------------------------- casts
_CAST_SRC = list(INT_BITS) + list(_FLOAT_PA) + [("dec", 9, 2), ("dec", 18, 0), ("dec", 38, 10), ("dec", 38, 0)]
_CAST_DST = list(INT_BITS) + list(_FLOAT_PA) + [("dec", 9, 2), ("dec", 18, 4), ("dec", 38, 10), ("dec", 38, 0), ("dec", 5, 0)]


def _src_values(t):
    if isinstance(t, tuple):
        p = t[1]
        big = [((2**53 + 1) << 64) + 2**63, (1 << 64) + 1, (1 << 64) - 1, 2**53 + 1, 10**20 + 5 * 10**9] if p == 38 else []
        half = [5 * 10 ** (t[2] - 1), -5 * 10 ** (t[2] - 1), 15 * 10 ** (t[2] - 1), 25 * 10 ** (t[2] - 1)] if t[2] > 0 else []
        return _dec_edges(p) + big + [-v for v in big] + half + _column(t, 300, 8)
    vals = edge_values(t) + _column(t, 300, 9)
    if t in _FLOAT_PA:   # values that round half away at the decimal targets' scales, and values at the int limits
        vals += [R.from_float(x, t) for x in (0.125, -0.125, 2.5, -2.5, 0.005, 127.5, -128.5, 2147483647.0, -2147483649.0, 9.2e18, 1e38, 1e-11)]
    return vals


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("src", _CAST_SRC, ids=str)
def test_casts_between_numeric_types(src, filtered):
    vals = _src_values(src) + [None]
    table = pa.table({"a": _arrow(vals, src), "id": pa.array(range(len(vals)), type=pa.int64())})
    dsts = [d for d in _CAST_DST if d != src]
    got, ids = _project(table, [P.try_cast(P.col("a"), _pa_type(d)) for d in dsts], dsts, filtered, True)
    _check(got, [lambda x, d=d: R.cast(x, src, d) for d in dsts], [(v,) for v in vals], ids, dsts, [f"{src}->{d}" for d in dsts])


# -------------------------------------------------------------------------------------------- decimals
# (op, lhs type, rhs type): the decimal matrix of TPC-DS money arithmetic, in the reference's plan shape
_DEC_CASES = [("Multiply", (38, 2), (10, 0)), ("Plus", (38, 2), (38, 2)), ("Multiply", (38, 10), (38, 10)), ("Multiply", (9, 2), (7, 4)),
              ("Minus", (18, 0), (18, 0)), ("Minus", (38, 2), (38, 2)), ("Plus", (9, 2), (18, 4))]


def _dec_operands(lt, rt):
    le, re_ = _dec_edges(lt[0]), _dec_edges(rt[0])
    a = [x for x in le + [None] for _ in re_ + [None]]
    b = [y for _ in le + [None] for y in re_ + [None]]
    # where a product or sum crosses 10^38 and 2^127
    a += [6 * 10**37, 10**37, 10**37, 5 * 10**36, 17 * 10**36, 85 * 10**35, 10**38 - 1, -(10**38 - 1), 10**38 // 2, 2**126 // 10**9]
    b += [2, 50, 17, 2, 10, 20, 1, -1, 10**38 // 2, 10**9]
    rng = random.Random(13)
    for _ in range(400):
        a.append(rng.randrange(-(10 ** lt[0]) + 1, 10 ** lt[0]) // 10 ** rng.randrange(0, lt[0]))
        b.append(rng.randrange(-(10 ** rt[0]) + 1, 10 ** rt[0]) // 10 ** rng.randrange(0, rt[0]))
    fit = lambda v, p: v if v is None or abs(v) < 10**p else (10**p - 1 if v > 0 else -(10**p - 1))
    return [fit(v, lt[0]) for v in a], [fit(v, rt[0]) for v in b]


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("op,lt,rt", _DEC_CASES, ids=lambda v: str(v))
def test_decimal_arithmetic_in_the_reference_plan_shape(op, lt, rt, filtered):
    a, b = _dec_operands(lt, rt)
    la, ra = ("dec",) + lt, ("dec",) + rt
    table = pa.table({"a": _arrow(a, la), "b": _arrow(b, ra), "id": pa.array(range(len(a)), type=pa.int64())})
    rp, rs = R.result_decimal_type(op, *lt, *rt)
    res = pa.decimal128(rp, rs)
    shaped = P.cast(P.binary(op, P.cast(P.col("a"), res), P.col("b")), res)
    ip, isc = R.engine_arith_type(op, *lt, *rt)
    raw = P.binary(op, P.col("a"), P.col("b"))                            # the bare operator, at the type the engine declares
    exprs = [shaped, raw, P.scalar_fn("Spark_CheckOverflow", [raw], res), P.cast(shaped, pa.float64())]
    types = [("dec", rp, rs), ("dec", ip, isc), ("dec", rp, rs), "float64"]
    fns = [lambda x, y: R.spark_decimal_op(op, x, *lt, y, *rt),
           lambda x, y: R.decimal_binary(op, x, lt[1], y, rt[1], ip),
           lambda x, y: R.check_overflow(R.decimal_binary(op, x, lt[1], y, rt[1], ip), isc, rp, rs),
           lambda x, y: R.cast(R.spark_decimal_op(op, x, *lt, y, *rt), ("dec", rp, rs), "float64")]
    got, ids = _project(table, exprs, types, filtered, False)
    _check(got, fns, list(zip(a, b)), ids, types, ["plan shape", "bare operator", "CheckOverflow", "as float64"])


@pytest.mark.parametrize("filtered", [False, True])
def test_decimal_functions(filtered):
    d = ("dec", 20, 8)
    vals = [12342132145623, 13245, 123213244568923, 1234567890, None, 10**20 - 1, -(10**20 - 1), 2**63, -(2**63) - 1, 2**64 + 5, 0,
            1, -1, 5 * 10**7, -5 * 10**7, 15 * 10**7, 25 * 10**7]
    ints = [12342132145623, 13245, 123213244568923, 1234567890, None, 10**10 - 1, 10**10, -(10**10), -(2**63), 2**63 - 1, 0, 1, -1, 99999,
            -99999, 100000, 5]
    table = pa.table({"d": _arrow(vals, d), "i": _arrow(ints, "int64"), "id": pa.array(range(len(vals)), type=pa.int64())})
    D, I = P.col("d"), P.col("i")
    exprs = [P.scalar_fn("Spark_CheckOverflow", [D], pa.decimal128(10, 5)), P.scalar_fn("Spark_CheckOverflow", [D], pa.decimal128(20, 8)),
             P.scalar_fn("Spark_CheckOverflow", [D], pa.decimal128(38, 10)), P.scalar_fn("Spark_CheckOverflow", [D], pa.decimal128(12, 0)),
             P.scalar_fn("Spark_MakeDecimal", [I], pa.decimal128(10, 5)), P.scalar_fn("Spark_MakeDecimal", [I], pa.decimal128(18, 2)),
             P.scalar_fn("Spark_UnscaledValue", [D], pa.int64()),
             P.scalar_fn("Spark_Round", [D, P.lit(0, pa.int32())], pa.decimal128(20, 8)),
             P.scalar_fn("Spark_BRound", [D, P.lit(0, pa.int32())], pa.decimal128(20, 8)),
             P.scalar_fn("Spark_Round", [I, P.lit(-1, pa.int32())], pa.int64()),
             P.scalar_fn("NullIf", [D, P.lit(decimal.Decimal("0.00013245"), pa.decimal128(20, 8))], pa.decimal128(20, 8)),
             P.scalar_fn("Spark_NullIfZero", [D], pa.decimal128(20, 8))]
    types = [("dec", 10, 5), ("dec", 20, 8), ("dec", 38, 10), ("dec", 12, 0), ("dec", 10, 5), ("dec", 18, 2), "int64", ("dec", 20, 8),
             ("dec", 20, 8), "int64", ("dec", 20, 8), ("dec", 20, 8)]
    fns = [lambda x, y: R.check_overflow(x, 8, 10, 5), lambda x, y: R.check_overflow(x, 8, 20, 8), lambda x, y: R.check_overflow(x, 8, 38, 10),
           lambda x, y: R.check_overflow(x, 8, 12, 0), lambda x, y: R.make_decimal(y, 10), lambda x, y: R.make_decimal(y, 18),
           lambda x, y: R.unscaled_value(x), lambda x, y: R.round_decimal(x, 8, 0), lambda x, y: R.round_decimal(x, 8, 0, half_even=True),
           lambda x, y: R.round_int(y, -1), lambda x, y: R.null_if(x, 13245), lambda x, y: R.null_if_zero(x, "dec")]
    got, ids = _project(table, exprs, types, filtered, False)
    _check(got, fns, list(zip(vals, ints)), ids, types,
           ["CheckOverflow(10,5)", "CheckOverflow(20,8)", "CheckOverflow(38,10)", "CheckOverflow(12,0)", "MakeDecimal(10,5)", "MakeDecimal(18,2)",
            "UnscaledValue", "Round", "BRound", "Round int", "NullIf", "NullIfZero"])


# -------------------------------------------------------------------------------------------- dates and strings
@pytest.mark.parametrize("filtered,hi", MODES)
def test_date_parts_and_date_text(filtered, hi):
    days = edge_values("date32") + [2932896, 2932897, -719162, -719163, -719528, -719529, 11016, 18321, -1, 59, 365, 366] + \
        [random.Random(6).randrange(-(1 << 31), 1 << 31) for _ in range(500)] + [None]
    table = pa.table({"d": pa.array(days, type=pa.int32()).cast(pa.date32()), "id": pa.array(range(len(days)), type=pa.int64())})
    dcol = P.col("d")
    parts = {"Spark_Year": "year", "Spark_Month": "month", "Spark_Day": "day", "Spark_Quarter": "quarter", "Spark_DayOfWeek": "dayofweek",
             "Spark_WeekOfYear": "week"}
    exprs = [P.scalar_fn(f, [dcol], pa.int32()) for f in parts] + \
        [P.scalar_fn("DatePart", [P.lit(p, pa.string()), dcol], pa.int32()) for p in ("dow", "doy", "quarter")] + \
        [P.try_cast(dcol, pa.string())]
    types = [pa.int32()] * (len(parts) + 3) + [pa.string()]
    fns = [lambda x, p=p: R.date_part(x, p) for p in parts.values()] + [lambda x, p=p: R.date_part(x, p) for p in ("dow", "doy", "quarter")] + \
        [R.date_text]
    got, ids = _project(table, exprs, types, filtered, hi)
    _check(got, fns, [(v,) for v in days], ids, types, list(parts) + ["dow", "doy", "date_part quarter", "date text"])


@pytest.mark.parametrize("filtered", [False, True])
def test_trim_case_and_octet_length(filtered):
    vals = [s.encode() for s in ["", " ", "  ", "a", " a", "a ", "  a b  ", "\ta\t", " é ", "ÿ", "aBc", "Straße", "\U0001F600 "]] + \
        [v for v in edge_values("utf8")] + [None]
    table = pa.table({"s": pa.array([None if v is None else v.decode() for v in vals]), "id": pa.array(range(len(vals)), type=pa.int64())})
    S = P.col("s")
    exprs = [P.scalar_fn(f, [S], pa.string()) for f in ("Trim", "Ltrim", "Rtrim", "Upper", "Lower")] + [P.scalar_fn("OctetLength", [S], pa.int32())]
    types = [pa.string()] * 5 + [pa.int32()]
    fns = [lambda x: R.trim(x), lambda x: R.trim(x, "left"), lambda x: R.trim(x, "right"), R.ascii_upper, R.ascii_lower, R.octet_length]
    got, ids = _project(table, exprs, types, filtered, False)
    _check(got, fns, [(v,) for v in vals], ids, types, ["Trim", "Ltrim", "Rtrim", "Upper", "Lower", "OctetLength"])


# -------------------------------------------------------------------------------------------- predicate fast paths
_PRED_TYPES = {"int8": pa.int8(), "int16": pa.int16(), "int32": pa.int32(), "int64": pa.int64(), "date32": pa.date32(), "date64": pa.date64(),
               "ts_s": pa.timestamp("s"), "ts_ms": pa.timestamp("ms"), "ts_us": pa.timestamp("us"), "ts_ns": pa.timestamp("ns"),
               "bool": pa.bool_(), "float32": pa.float32(), "float64": pa.float64(), "dec9_2": pa.decimal128(9, 2), "dec38_10": pa.decimal128(38, 10)}


def _pred_column(t, n):
    if t in ("date32", "date64") or t.startswith("ts_"):
        vals = edge_values(t) + [v for v in _column("int32", n, 21)]
        vals = [None if v is None else (v * 86_400_000 if t == "date64" and abs(v) < 2**31 else v) for v in vals]
        return vals, pa.array(vals, type=pa.int64() if t != "date32" else pa.int32()).cast(_PRED_TYPES[t])
    if t == "bool":
        vals = [None, True, False] * (n // 3)
        return vals, pa.array(vals)
    if t.startswith("dec"):
        dt = ("dec", _PRED_TYPES[t].precision, _PRED_TYPES[t].scale)
        vals = _column(dt, n, 22)
        return vals, _arrow(vals, dt)
    vals = edge_values(t) + _column(t, n, 23)
    return vals, _arrow(vals, t)


def _pred_literals(t):
    """(literal value as Python, literal pa type, canonical value) at and beyond the column type's range"""
    if t in INT_BITS:
        b = INT_BITS[t]
        lo, hi = -(1 << (b - 1)), (1 << (b - 1)) - 1
        out = [(v, _PRED_TYPES[t], v) for v in (lo, hi, 0, -1)]
        if b < 64:
            out += [(v, pa.int64(), v) for v in (lo - 1, hi + 1, -(2**63), 2**63 - 1)]
        return out
    if t == "date32":
        return [(v, pa.int32(), v) for v in (-(2**31), 2**31 - 1, 0)]
    if t == "date64":
        return [(v, pa.int64(), v) for v in (-(2**63), 2**63 - 1, 0, 86_400_000)]
    if t.startswith("ts_"):
        return [(v, _PRED_TYPES[t], v) for v in (-(2**63), 2**63 - 1, 0, -1)]
    if t == "bool":
        return [(True, pa.bool_(), True), (False, pa.bool_(), False)]
    if t in _FLOAT_PA:
        return [(R.to_float(v, t), _FLOAT_PA[t], v) for v in (0, 1 << (31 if t == "float32" else 63), R.from_float(float("nan"), t),
                                                              R.from_float(float("inf"), t), R.from_float(1.0, t))]
    dt = _PRED_TYPES[t]
    m = 10 ** dt.precision - 1
    return [(unscaled_to_decimal(v, dt.scale), dt, v) for v in (m, -m, 0, 1)]


def _filter_rows(table, preds, vm: bool):
    if vm:
        os.environ["AURON_DISABLE_SIMPLE_PREDICATE"] = "1"
    try:
        return run(P.filter_(P.ffi_reader(table.schema, "t"), preds), {"t": table})["id"].to_pylist()
    finally:
        os.environ.pop("AURON_DISABLE_SIMPLE_PREDICATE", None)


@pytest.mark.parametrize("t", list(_PRED_TYPES))
def test_predicate_fast_paths_match_vm_and_reference(t):
    vals, arr = _pred_column(t, 3000)
    table = pa.table({"c": arr, "id": pa.array(range(len(vals)), type=pa.int64())})
    ct = t if t in _FLOAT_PA else "int"
    for lit, lty, canon in _pred_literals(t):
        runs = [(op, False, []) for op in ("Eq", "NotEq", "Lt", "LtEq", "Gt", "GtEq")] + [("Lt", True, []), ("GtEq", True, [])] + \
            [("LtEq", False, [P.is_not_null(P.col("c")), P.binary("GtEq", P.col("id"), P.lit(7, pa.int64()))])]
        for op, mirrored, extra in runs:   # column <op> literal, literal <op> column, and the term among others
            term = P.binary(op, P.lit(lit, lty), P.col("c")) if mirrored else P.binary(op, P.col("c"), P.lit(lit, lty))
            fast = _filter_rows(table, [term] + extra, vm=False)
            vm = _filter_rows(table, [term] + extra, vm=True)
            exp = [i for i, v in enumerate(vals) if (R.compare(op, canon, v, ct) if mirrored else R.compare(op, v, canon, ct)) and (not extra or i >= 7)]
            assert fast == vm, (t, lit, op, mirrored, len(extra))
            assert fast == exp, (t, lit, op, mirrored, len(extra))
    for fn, neg in (("is_null", False), ("is_not_null", True)):
        e = getattr(P, fn)(P.col("c"))
        assert _filter_rows(table, [e], False) == _filter_rows(table, [e], True) == [i for i, v in enumerate(vals) if (v is not None) == neg]


@pytest.mark.parametrize("unit,other", [("ms", "s"), ("us", "ns"), ("s", "ns"), ("ns", "ms")])
def test_predicate_on_timestamps_of_another_unit_is_rejected_on_both_paths(unit, other):
    # a literal of another unit means another instant for the same raw number: neither path may compare the raw numbers
    table = pa.table({"c": pa.array([0, 1, 1000, -1], type=pa.int64()).cast(pa.timestamp(unit)), "id": pa.array(range(4), type=pa.int64())})
    preds = [P.binary("Gt", P.col("c"), P.lit(1, pa.timestamp(other)))]
    for vm in (True, False):
        with pytest.raises(runtime.AuronError, match="timestamps of different units"):
            _filter_rows(table, preds, vm)
