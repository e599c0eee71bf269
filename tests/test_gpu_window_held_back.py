"""WindowExec's held-back rows and its 128-bit running sum, on device batches of a prime number of rows (AURON_GPU_CHUNK_ROWS).

* When a function needs the whole partition (LEAD, window/mod.rs:115-120), the open partition is held back and put in front of the next
  batch.  The held-back batches are kept as they are and concatenated once, when their partition closes or the input ends
  (window_exec.rs:227-291): the operator's `concat_rows` metric counts the rows it copied that way, at most every row once.
* A window SUM over decimal128 wraps on i128 overflow, as the reference's accumulator does (agg/sum.rs:115).
"""
import decimal

import numpy as np
import pyarrow as pa
import pytest

import oracle
from auron_b200 import proto as P
from auron_b200 import runtime

pytestmark = pytest.mark.gpu

CHUNK = 7_919
I, L = pa.int32(), pa.int64()


@pytest.fixture
def prime_batches(monkeypatch):
    monkeypatch.setenv("AURON_GPU_CHUNK_ROWS", str(CHUNK))


def _table(sizes, seed):
    rng = np.random.default_rng(seed)
    p = np.repeat(np.arange(len(sizes), dtype=np.int32), sizes)
    o = np.concatenate([np.sort(rng.integers(0, max(2, s // 4), s)) for s in sizes]).astype(np.int64)
    n = len(p)
    return pa.table({"p": pa.array(p), "o": pa.array(o), "v": pa.array(rng.integers(-1000, 1000, n), type=L, mask=rng.random(n) < 0.1)})


def _run_with_metrics(plan, t):
    with runtime.Task(P.task_definition(plan), {"t": t.to_batches(max_chunksize=CHUNK)}) as task:
        out = pa.Table.from_batches(list(task), schema=task.schema)
        m = task.metrics()
    return out, sum(v for _, op, name, v in m if op == "WindowExec" and name == "concat_rows")


def _lead(t, partition):
    wex = [P.window_expr("rn", I, "ROW_NUMBER"), P.window_expr("ld", L, "LEAD", [P.col("v"), P.lit(1, I), P.lit(None, L)])]
    return P.window(P.ffi_reader(t.schema, "t"), wex, [P.col("p")] if partition else [], [P.sort_expr(P.col("o"))])


@pytest.mark.parametrize("partition", [False, True])
def test_held_back_rows_are_copied_once(prime_batches, partition):
    # small partitions around one of 70,000 rows (9 batches): without a partition spec the whole input is held back and concatenated
    # once at the end; with one, only the batches of the open partition are, each row at most once
    sizes = [3] * 2000 + [70_000] + [5] * 2000
    t = _table(sizes, 7)
    n = t.num_rows
    got, copied = _run_with_metrics(_lead(t, partition), t)
    assert got.num_rows == n
    rows = list(zip(*[got[c].to_pylist() for c in ("p", "o", "v")]))
    assert rows == list(zip(*[t[c].to_pylist() for c in ("p", "o", "v")]))
    exp = oracle.window_functions(rows, (lambda r: r[0]) if partition else (lambda r: 0), lambda r: r[1],
                                  [("ROW_NUMBER", None, None), ("LEAD", lambda r: r[2], (1, lambda r: None))])
    assert list(zip(got["rn"].to_pylist(), got["ld"].to_pylist())) == exp
    if partition:
        assert 70_000 <= copied <= n      # the long partition's batches are joined once; batches closed inside themselves are not copied
    else:
        assert copied == n


def _i128(col):
    """unscaled values of a decimal128 column read from its buffer (also those beyond its declared precision)"""
    arr = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    words = np.frombuffer(arr.buffers()[1], dtype=np.int64)[2 * arr.offset:2 * (arr.offset + len(arr))].reshape(-1, 2)
    valid = arr.is_valid().to_pylist()
    return [((int(lo) & (2**64 - 1)) | (int(hi) << 64)) if ok else None for (lo, hi), ok in zip(words, valid)]


def _wrap128(x):
    x &= (1 << 128) - 1
    return x - (1 << 128) if x >> 127 else x


def test_decimal_sum_wraps_at_128_bits(prime_batches):
    # decimal(38,0) values near +-10^38 in a partition of 20,000 rows (three batch edges): the running sum leaves the i128 range again and
    # again and wraps; a saturating or overflow-to-NULL sum would differ
    rng = np.random.default_rng(127)
    sizes = [20_000, 3, 7_000]
    n = sum(sizes)
    p = np.repeat(np.arange(len(sizes), dtype=np.int32), sizes)
    big = [int(a) * 10**20 + int(b) for a, b in zip(rng.integers(-10**18 + 1, 10**18, n), rng.integers(0, 2**62, n))]
    big[:4] = [10**38 - 1] * 4
    mask = rng.random(n) < 0.05
    mask[:4] = False
    dec = pa.decimal128(38, 0)
    t = pa.table({"p": pa.array(p), "o": pa.array(np.arange(n, dtype=np.int64)),
                  "d": pa.array([None if mask[i] else decimal.Decimal(big[i]) for i in range(n)], type=dec)})
    plan = P.window(P.ffi_reader(t.schema, "t"), [P.window_expr("s", dec, "SUM", [P.col("d")])], [P.col("p")], [P.sort_expr(P.col("o"))])
    got = runtime.run_task(P.task_definition(plan), {"t": t.to_batches(max_chunksize=CHUNK)})
    exp, acc, prev = [], None, None
    for i in range(n):
        if p[i] != prev:
            prev, acc = p[i], None
        if not mask[i]:
            acc = big[i] if acc is None else _wrap128(acc + big[i])
        exp.append(acc)
    assert exp[1] == _wrap128(2 * (10**38 - 1)) and exp[1] < 0     # the second row already wraps
    assert sum(1 for a, b in zip(exp, exp[1:]) if a is not None and b is not None and (a > 0) != (b > 0)) > 100
    assert _i128(got["s"]) == exp
