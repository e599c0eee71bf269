"""Plain-Python references for the key semantics of sort, grouping, join and partitioning, and the edge values of every key type.

Values are kept in one canonical form per type, so that the references never go through a float conversion or a library:
  * integers, date32 / date64 and timestamps: the Python int that is stored,
  * float32 / float64: the IEEE bit pattern as an unsigned int (NaN payloads and the sign of zero survive),
  * decimals: the unscaled integer,
  * bool: a Python bool,
  * utf8 / binary: bytes,
  * NULL: None.
Only Python ints, `decimal`, `struct` and bytes are used here -- no engine, no numpy, no Arrow."""
from __future__ import annotations

import bisect
import decimal
import functools
import random
import struct

SENTINEL = 0x8A5C3F1E9D7B2461                       # the empty-slot marker of the aggregate and join hash tables
SENTINEL_I64 = SENTINEL - (1 << 64)                 # ... read as a signed int64

RADIX_TILE = 4096                                   # rows per tile of the radix sort (k_sort.cu RS_TILE)
DAY_MS = 86_400_000                                 # date64 holds milliseconds of whole days
SCAN_BLOCK = 2048                                   # elements per block of the device scans

INT_BITS = {"int8": 8, "int16": 16, "int32": 32, "int64": 64}
TIMESTAMPS = ("ts_s", "ts_ms", "ts_us", "ts_ns")
DECIMALS = {"dec9_2": (9, 2), "dec18_0": (18, 0), "dec38_10": (38, 10)}
FLOATS = ("float32", "float64")
TYPES = tuple(INT_BITS) + FLOATS + ("bool", "date32", "date64") + TIMESTAMPS + tuple(DECIMALS) + ("utf8", "binary")
FIXED_WIDTH = tuple(t for t in TYPES if t not in ("utf8", "binary"))


def f32_bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def bits_f32(b: int) -> float:
    return struct.unpack("<f", struct.pack("<I", b))[0]


def _float_edges(bits: int) -> list[int]:
    sign = 1 << (bits - 1)
    exp_bits = 8 if bits == 32 else 11
    mant = bits - 1 - exp_bits
    inf = ((1 << exp_bits) - 1) << mant
    quiet = inf | (1 << (mant - 1))
    one = f32_bits(1.0) if bits == 32 else f64_bits(1.0)
    return [0, sign,                                   # +0.0, -0.0
            inf, sign | inf,                           # +inf, -inf
            quiet, sign | quiet,                       # canonical quiet NaN, with the sign bit clear and set
            quiet | 0x2345,                            # a NaN with another payload
            1,                                         # smallest subnormal
            inf - 1,                                   # largest finite
            one, sign | one]                           # +1, -1


_STR_EDGES = ["", "\x00", "a", "a\x00"] + [p + c for n in (7, 8, 9, 15, 16, 17, 64) for p in ["q" * (n - 1)] for c in "ab"] + \
             ["é", "ÿ", "aé", "\U0001F600", "\U0001F600\U0001F600"]


def edge_values(t: str) -> list:
    """The edge set of type t, in canonical form."""
    if t in INT_BITS:
        b = INT_BITS[t]
        lo, hi = -(1 << (b - 1)), (1 << (b - 1)) - 1
        vals = [lo, lo + 1, -1, 0, 1, hi - 1, hi]
        return vals + ([SENTINEL_I64] if t == "int64" else [])
    if t == "float32":
        return _float_edges(32)
    if t == "float64":
        return _float_edges(64) + [SENTINEL]
    if t == "bool":
        return [False, True]
    if t == "date32":
        return [-(1 << 31), (1 << 31) - 1, -1, 0, 1]
    if t == "date64":                                  # milliseconds of whole days
        return [-(2 ** 63 // DAY_MS) * DAY_MS, (2 ** 63 - 1) // DAY_MS * DAY_MS, -DAY_MS, 0, DAY_MS]
    if t in TIMESTAMPS:
        return [-(1 << 63), (1 << 63) - 1, -1, 0, 1]
    if t in ("dec9_2", "dec18_0"):
        m = 10 ** DECIMALS[t][0] - 1
        return [m, -m, 1, -1, 0]
    if t == "dec38_10":
        m, w = 10 ** 38 - 1, 1 << 64
        # 1, 1 + 2^64, 1 + 2^65 and 1 - 2^64 share their low 64-bit word and differ only in the high one
        return [m, -m, w, -w, w - 1, -(w - 1), -1, 0, 1 + w, 1 + 2 * w]
    if t == "utf8":
        return [s.encode() for s in _STR_EDGES]
    if t == "binary":
        return [s.encode() for s in _STR_EDGES] + [b"\xff", b"\xff" * 8, b"\xff" * 9, b"\xff" * 17, b"a\xff"]
    raise ValueError(t)


def _random_value(t: str, rng: random.Random):
    if t in INT_BITS:
        b = INT_BITS[t]
        return rng.randrange(-(1 << (b - 1)), 1 << (b - 1))
    if t == "float32":
        return f32_bits(rng.uniform(-1e6, 1e6))
    if t == "float64":
        return f64_bits(rng.uniform(-1e12, 1e12))
    if t == "bool":
        return rng.random() < 0.5
    if t == "date32":
        return rng.randrange(-50_000, 50_000)
    if t == "date64":
        return rng.randrange(-(1 << 36), 1 << 36) * DAY_MS
    if t in TIMESTAMPS:
        return rng.randrange(-(1 << 62), 1 << 62)
    if t in DECIMALS:
        m = 10 ** DECIMALS[t][0] - 1
        return rng.randrange(-m, m + 1)
    if t in ("utf8", "binary"):
        return "".join(rng.choice("pqaé") for _ in range(rng.randrange(0, 20))).encode()
    raise ValueError(t)


def edge_column(t: str, n: int, seed: int, rate: float = 0.2, null_rate: float = 0.05) -> list:
    """n values of type t: random fill, every edge value mixed in at `rate`, and the edge values (and a NULL, when null_rate > 0)
    written on both sides of every scan block / radix tile boundary below n.  Deterministic per seed."""
    rng = random.Random(seed)
    edges = edge_values(t)
    out = []
    for _ in range(n):
        u = rng.random()
        if u < null_rate:
            out.append(None)
        elif u < null_rate + rate:
            out.append(rng.choice(edges))
        else:
            out.append(_random_value(t, rng))
    special = edges + ([None] if null_rate > 0 else [])
    k = rng.randrange(len(special))
    for b in range(SCAN_BLOCK, n, SCAN_BLOCK):          # every other boundary is also a radix tile boundary
        for pos in (b - 2, b - 1, b, b + 1):
            if 0 <= pos < n:
                out[pos] = special[k % len(special)]
                k += 1
    for i, v in enumerate(special):                      # every value at least once, also when n is small
        out[(i * 7919 + seed) % n] = v
    return out


# -------------------------------------------------------------------------------------------- order (arrow-row, sort_exec.rs)
@functools.total_ordering
class _Desc:
    """reverses the order of a wrapped value (descending keys of any type, bytes included)"""
    __slots__ = ("v",)

    def __init__(self, v):
        self.v = v

    def __eq__(self, o):
        return self.v == o.v

    def __lt__(self, o):
        return o.v < self.v


def total_order(bits: int, width: int) -> int:
    """IEEE totalOrder of a float bit pattern as a signed int: -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN"""
    sign = bits >> (width - 1)
    magnitude = bits & ((1 << (width - 1)) - 1)
    return -magnitude - 1 if sign else magnitude


def value_order(v, t: str):
    """order key of a non-NULL value of type t (ascending)"""
    if t in FLOATS:
        return total_order(v, 32 if t == "float32" else 64)
    if t == "bool":
        return int(v)
    return v                                             # ints, dates, timestamps, unscaled decimals, bytes (unsigned bytewise)


def sort_key(value, t: str, asc: bool = True, nulls_first: bool = True):
    """the position of one value in the reference's sort order for one key (arrow-row encoding)"""
    if value is None:
        return (0 if nulls_first else 2, 0)
    k = value_order(value, t)
    return (1, k if asc else _Desc(k))


def row_sort_key(row, specs):
    """row = tuple of values; specs = [(type, asc, nulls_first)] for every key"""
    return tuple(sort_key(v, t, a, nf) for v, (t, a, nf) in zip(row, specs))


def range_partition_ids(keys, bounds, specs):
    """range partitioning: the number of bounds strictly below the row's key (bisect_left in sort_key order)"""
    bk = [row_sort_key(b, specs) for b in bounds]
    return [bisect.bisect_left(bk, row_sort_key(k, specs)) for k in keys]


# -------------------------------------------------------------------------------------------- grouping and accumulators
def group_rows(keys) -> dict:
    """group key tuple -> row indices in input order.  Canonical values already compare floats by their bits; NULL is a group."""
    groups: dict = {}
    for i, k in enumerate(keys):
        groups.setdefault(k, []).append(i)
    return groups


def wrap(v: int, bits: int) -> int:
    """two's-complement wrap of an exact integer to `bits` bits"""
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def wrapping_sum(values, bits: int = 64):
    """SUM of the non-NULL values, wrapping at 2^bits (int64: 64, decimal128: 128); NULL when every value is NULL"""
    vals = [v for v in values if v is not None]
    return wrap(sum(vals), bits) if vals else None


def div_euclid(a: int, b: int) -> int:
    """Rust's i128::div_euclid: the quotient whose remainder is never negative"""
    q, r = divmod(a, b)                                  # Python's remainder has the sign of b
    if r < 0:
        q, r = q + 1, r - b
    return q


def decimal_avg(values):
    """AVG over decimals at the argument's scale (avg_finalize): div_euclid of the wrapped i128 sum by the count"""
    vals = [v for v in values if v is not None]
    return div_euclid(wrap(sum(vals), 128), len(vals)) if vals else None


def extreme(values, t: str, want_max: bool):
    """MIN / MAX of the non-NULL values in the engine's total order (floats: IEEE totalOrder, so NaN > +inf and
    MIN(-0.0, +0.0) = -0.0); NULL when every value is NULL"""
    vals = [v for v in values if v is not None]
    if not vals:
        return None
    return (max if want_max else min)(vals, key=lambda v: value_order(v, t))


# -------------------------------------------------------------------------------------------- joins
def join_rows(lkeys, rkeys, how: str):
    """Equi-join of two lists of key tuples: NULL never matches, everything else (floats by their bits) matches on equality.
    Returns the sorted (left row, right row) pairs of the result, None for the missing side; SEMI / ANTI give (left row, None)."""
    index: dict = {}
    for j, k in enumerate(rkeys):
        if None not in k:
            index.setdefault(k, []).append(j)
    out, right_hit = [], set()
    for i, k in enumerate(lkeys):
        m = [] if None in k else index.get(k, [])
        if how == "SEMI":
            out += [(i, None)] if m else []
        elif how == "ANTI":
            out += [] if m else [(i, None)]
        else:
            out += [(i, j) for j in m]
            right_hit.update(m)
            if not m and how in ("LEFT", "FULL"):
                out.append((i, None))
    if how in ("RIGHT", "FULL"):
        out += [(None, j) for j in range(len(rkeys)) if j not in right_hit]
    return sorted(out, key=lambda p: (p[0] is None, p[0] or 0, p[1] is None, p[1] or 0))


# -------------------------------------------------------------------------------------------- decimals as Python Decimals
def unscaled_to_decimal(v: int, scale: int) -> decimal.Decimal:
    return decimal.Decimal(v).scaleb(-scale, decimal.Context(prec=60))
