"""WindowExec batch by batch (window_exec.rs:206-306): pre-sorted input fed through ffi_reader in device batches of a prime number of
rows (AURON_GPU_CHUNK_ROWS), so batch edges fall inside partitions and peer groups.  The running functions carry their state across
every edge; functions that need the whole partition (LEAD) hold back the open partition.  Window aggregates over decimals, strings,
binary, booleans, timestamps and date64 are checked against the reference's accumulators restated on Python values
(agg/sum.rs, avg.rs, maxmin.rs)."""
import decimal
import os
import sys

import numpy as np
import pyarrow as pa
import pytest

import oracle
from auron_b200 import proto as P
from auron_b200 import runtime

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tpcds_replay as R  # noqa: E402

pytestmark = pytest.mark.gpu

CHUNK = 7_919          # a prime: device batches end at arbitrary rows
I, L, F, S = pa.int32(), pa.int64(), pa.float64(), pa.string()
D = decimal.Decimal
CTX = decimal.Context(prec=80)   # exact scaling of 38-digit values


@pytest.fixture
def prime_batches(monkeypatch):
    monkeypatch.setenv("AURON_GPU_CHUNK_ROWS", str(CHUNK))   # read when the task's context is created


def _layout(seed):
    """(partition key, order key) rows in window order: partitions of 1 and 4 rows, ~1000 rows, one of 60,000 rows (more than 5
    batches) whose order key runs in peer groups of 3,000 rows (crossing batch edges), a NULL partition key and NULL order keys"""
    rng = np.random.default_rng(seed)
    sizes = [1] * 300 + [4] * 300 + [int(x) for x in rng.integers(500, 1500, 20)] + [1] * 50 + [int(x) for x in rng.integers(2, 40, 200)]
    rng.shuffle(sizes)
    sizes.insert(len(sizes) // 2, 60_000)
    rows = []
    for k in range(len(sizes) + 1):
        size = int(sizes[k]) if k < len(sizes) else 700
        p = None if k == len(sizes) else k          # the NULL partition: a group of its own
        if size >= 60_000:
            orders = [j // 3_000 for j in range(size)]
        else:
            orders = sorted(int(x) for x in rng.integers(0, max(2, size // 3), size))
        n_null = int(rng.integers(0, 3)) if size > 3 else 0
        rows += [(p, None if j < n_null else o) for j, o in enumerate(orders)]
    return rows, rng


def _batches(t: pa.Table, chunk=CHUNK):
    return t.combine_chunks().to_batches(max_chunksize=chunk)


def _run(plan, t: pa.Table, chunk=CHUNK):
    return runtime.run_task(P.task_definition(plan, stage_id=1, partition_id=0, task_id=7), {"t": _batches(t, chunk)})


def _window(t, wex, group_limit=None, output_window_cols=True, partition=True):
    return P.window(P.ffi_reader(t.schema, "t"), wex, [P.col("p")] if partition else [], [P.sort_expr(P.col("o"))], group_limit=group_limit,
                    output_window_cols=output_window_cols)


def _cols(t, names):
    return list(zip(*[t[c].to_pylist() for c in names]))


def test_running_functions_across_batch_edges(prime_batches, monkeypatch):
    keys, rng = _layout(1)
    n = len(keys)
    t = pa.table({"p": pa.array([k[0] for k in keys], type=I), "o": pa.array([k[1] for k in keys], type=L),
                  "v": pa.array(rng.integers(-1000, 1000, n), type=L, mask=rng.random(n) < 0.1),
                  "f": pa.array(np.round(rng.standard_normal(n), 3), mask=rng.random(n) < 0.1)})
    wex = [P.window_expr("rn", I, "ROW_NUMBER"), P.window_expr("rk", I, "RANK"), P.window_expr("dr", I, "DENSE_RANK"),
           P.window_expr("nth", L, "NTH_VALUE", [P.col("v"), P.lit(3, I)]), P.window_expr("nthn", L, "NTH_VALUE_IGNORE_NULLS", [P.col("v"), P.lit(2, I)]),
           P.window_expr("sv", L, "SUM", [P.col("v")]), P.window_expr("cv", L, "COUNT", [P.col("v")]), P.window_expr("mn", L, "MIN", [P.col("v")]),
           P.window_expr("mx", L, "MAX", [P.col("v")]), P.window_expr("sf", F, "SUM", [P.col("f")]), P.window_expr("cf", L, "COUNT", [P.col("f")]),
           P.window_expr("mnf", F, "MIN", [P.col("f")]), P.window_expr("mxf", F, "MAX", [P.col("f")]), P.window_expr("av", F, "AVG", [P.col("v")]),
           P.window_expr("avf", F, "AVG", [P.col("f")])]
    names = ["rn", "rk", "dr", "nth", "nthn", "sv", "cv", "mn", "mx", "sf", "cf", "mnf", "mxf", "av", "avf"]
    got = _run(_window(t, wex), t)
    assert n > 10 * CHUNK and got.num_rows == n
    rows = _cols(got, ["p", "o", "v", "f"])
    assert rows == _cols(t, ["p", "o", "v", "f"])                        # input order
    v_of, f_of = (lambda r: r[2]), (lambda r: r[3])
    exp = oracle.window_functions(rows, lambda r: r[0], lambda r: r[1],
                                  [("ROW_NUMBER", None, None), ("RANK", None, None), ("DENSE_RANK", None, None), ("NTH_VALUE", v_of, 3),
                                   ("NTH_VALUE_IGNORE_NULLS", v_of, 2), ("SUM", v_of, None), ("COUNT", v_of, None), ("MIN", v_of, None), ("MAX", v_of, None),
                                   ("SUM", f_of, None), ("COUNT", f_of, None), ("MIN", f_of, None), ("MAX", f_of, None), ("AVG", v_of, None),
                                   ("AVG", f_of, None)])
    out = _cols(got, names)
    for i, (g, e) in enumerate(zip(out, exp)):
        assert g[:9] == e[:9] and g[10:13] == e[10:13], (i, rows[i], g, e)
        for a, b in (g[9], e[9]), (g[13], e[13]), (g[14], e[14]):       # float sums: scan order differs from row order
            assert (a is None) == (b is None) and (a is None or abs(a - b) <= 1e-6 * max(1.0, abs(b))), (i, g, e)
    # the integer outputs are bit-identical to one batch over the whole input
    monkeypatch.delenv("AURON_GPU_CHUNK_ROWS")
    whole = _run(_window(t, wex), t, chunk=n)
    ints = ["rn", "rk", "dr", "nth", "nthn", "sv", "cv", "mn", "mx", "cf"]
    assert _cols(whole, ints) == _cols(got, ints)


def _unscaled(d, scale):
    return None if d is None else int(d.scaleb(scale, context=CTX))


def _wrap128(x):
    x &= (1 << 128) - 1
    return x - (1 << 128) if x >> 127 else x


def _running(rows, part_of, arg_of, step):
    """the accumulator after every row, reset at partition changes; NULL arguments skipped, NULL until the first value"""
    out, prev, acc = [], object(), None
    for r in rows:
        if part_of(r) != prev:
            prev, acc = part_of(r), None
        v = arg_of(r)
        if v is not None:
            acc = v if acc is None else step(acc, v)
        out.append(acc)
    return out


def test_decimal_aggregates_across_batch_edges(prime_batches):
    keys, rng = _layout(2)
    n = len(keys)
    cents = rng.integers(-10**12, 10**12, n)
    big = [int(x) * 10**20 + int(y) for x, y in zip(rng.integers(-10**8, 10**8, n), rng.integers(0, 10**12, n))]   # beyond 64 bits
    null17, null38 = rng.random(n) < 0.1, rng.random(n) < 0.1
    # the NULL partition holds small negative values: AVG must round toward negative infinity (div_euclid)
    d17 = [None if null17[i] else (D(-1 - i % 3) if keys[i][0] is None else D(int(cents[i]))).scaleb(-2, context=CTX) for i in range(n)]
    t = pa.table({"p": pa.array([k[0] for k in keys], type=I), "o": pa.array([k[1] for k in keys], type=L),
                  "d17": pa.array(d17, type=pa.decimal128(17, 2)),
                  "d38": pa.array([None if null38[i] else D(big[i]).scaleb(-10, context=CTX) for i in range(n)], type=pa.decimal128(38, 10))})
    dec27, dec21, dec17, dec38 = pa.decimal128(27, 2), pa.decimal128(21, 6), pa.decimal128(17, 2), pa.decimal128(38, 10)
    wex = [P.window_expr("s", dec27, "SUM", [P.col("d17")]), P.window_expr("a", dec21, "AVG", [P.col("d17")]),
           P.window_expr("mn", dec17, "MIN", [P.col("d17")]), P.window_expr("mx", dec17, "MAX", [P.col("d17")]),
           P.window_expr("mn38", dec38, "MIN", [P.col("d38")]), P.window_expr("mx38", dec38, "MAX", [P.col("d38")])]
    got = _run(_window(t, wex), t)
    assert got.schema.field("s").type == dec27 and got.schema.field("a").type == dec21
    rows = [(p, o, _unscaled(a, 2), _unscaled(b, 10)) for p, o, a, b in _cols(got, ["p", "o", "d17", "d38"])]
    assert [r[:2] for r in rows] == keys
    part = lambda r: r[0]
    exp_s = _running(rows, part, lambda r: r[2], lambda a, b: _wrap128(a + b))
    # AVG: TryCast(decimal(17,2) -> decimal(21,6)) = unscaled * 10^4, then a running i128 sum and count, sum.div_euclid(count)
    sums = _running(rows, part, lambda r: None if r[2] is None else r[2] * 10**4, lambda a, b: _wrap128(a + b))
    counts = _running(rows, part, lambda r: None if r[2] is None else 1, lambda a, b: a + b)
    exp_a = [None if c is None else s // c for s, c in zip(sums, counts)]   # count > 0: floor == euclid
    exp = list(zip(exp_s, exp_a, _running(rows, part, lambda r: r[2], min), _running(rows, part, lambda r: r[2], max),
                   _running(rows, part, lambda r: r[3], min), _running(rows, part, lambda r: r[3], max)))
    g = [(_unscaled(s, 2), _unscaled(a, 6), _unscaled(mn, 2), _unscaled(mx, 2), _unscaled(m38, 10), _unscaled(x38, 10))
         for s, a, mn, mx, m38, x38 in _cols(got, ["s", "a", "mn", "mx", "mn38", "mx38"])]
    for i, (gi, ei) in enumerate(zip(g, exp)):
        assert gi == ei, (i, rows[i], gi, ei)
    assert any(c is not None and s < 0 and s % c for s, c in zip(sums, counts))          # inexact negative averages: floor, not truncation
    assert any(e[5] is not None and abs(e[5]) >= 1 << 64 for e in exp)


def _strings(rng, n):
    words = ["", "a", "ab", "abc", "abd", "b", "é", "éa", "日本", "日本語", "z" * 2048, "z" * 2047, "\x00", "zz"]
    return [None if rng.random() < 0.1 else words[int(rng.integers(0, len(words)))] + ("" if rng.random() < 0.7 else str(int(rng.integers(0, 50))))
            for _ in range(n)]


def test_string_binary_bool_and_time_extremes_across_batch_edges(prime_batches):
    keys, rng = _layout(3)
    n = len(keys)
    s = _strings(rng, n)
    ts = rng.integers(-10**15, 10**15, n)
    d64 = rng.integers(-10**5, 10**5, n) * 86_400_000
    t = pa.table({"p": pa.array([k[0] for k in keys], type=I), "o": pa.array([k[1] for k in keys], type=L), "s": pa.array(s, type=S),
                  "b": pa.array([None if x is None else x.encode()[::-1] for x in s], type=pa.binary()),
                  "f": pa.array([None if rng.random() < 0.1 else bool(rng.random() < 0.5) for _ in range(n)], type=pa.bool_()),
                  "ts": pa.array(ts, type=pa.timestamp("us"), mask=rng.random(n) < 0.1),
                  "tn": pa.array(ts, type=pa.timestamp("ns", tz="UTC"), mask=rng.random(n) < 0.1),
                  "d64": pa.array(d64, type=pa.date64(), mask=rng.random(n) < 0.1)})
    cols = ["s", "b", "f", "ts", "tn", "d64"]
    wex, names = [], []
    for c in cols:
        for fn in ("MIN", "MAX"):
            wex.append(P.window_expr(f"{fn}_{c}", t.schema.field(c).type, fn, [P.col(c)]))
            names.append(f"{fn}_{c}")
    got = _run(_window(t, wex), t)
    for c in cols:
        assert got.schema.field(f"MIN_{c}").type == t.schema.field(c).type
    # utf8 compares byte-wise: encode before comparing (Python's str order is by code point, which UTF-8 bytes preserve anyway)
    ints = {"ts": t["ts"].cast(L).to_pylist(), "tn": t["tn"].cast(L).to_pylist(), "d64": t["d64"].cast(L).to_pylist()}
    vals = {"s": [None if x is None else x.encode() for x in s], "b": t["b"].to_pylist(), "f": t["f"].to_pylist(), **ints}
    rows = list(range(n))
    part = lambda i: keys[i][0]
    for c in cols:
        got_c = {fn: got[f"{fn}_{c}"] for fn in ("MIN", "MAX")}
        for fn, agg in (("MIN", min), ("MAX", max)):
            exp = _running(rows, part, lambda i: vals[c][i], agg)
            g = got_c[fn]
            g = [None if x is None else x.encode() for x in g.to_pylist()] if c == "s" else (g.cast(L).to_pylist() if c in ints else g.to_pylist())
            bad = [i for i in range(n) if g[i] != exp[i]]
            assert not bad, (c, fn, bad[:5], [(g[i], exp[i]) for i in bad[:3]])


class _Recorder:
    """input batches handed out one at a time; pulled[k] = input batches pulled when output batch k arrived"""

    def __init__(self, batches):
        self.batches, self.n = batches, 0

    def __iter__(self):
        for b in self.batches:
            self.n += 1
            yield b


def _stream(plan, t):
    rec = _Recorder(_batches(t))
    pulled, out = [], []
    with runtime.Task(P.task_definition(plan), {"t": rec}) as task:
        for b in task:
            pulled.append(rec.n)
            out.append(b)
    return pa.Table.from_batches(out, schema=task.schema), pulled, len(rec.batches)


def test_batches_stream_through(prime_batches):
    keys, rng = _layout(4)
    n = len(keys)
    t = pa.table({"p": pa.array([k[0] for k in keys], type=I), "o": pa.array([k[1] for k in keys], type=L),
                  "v": pa.array(rng.integers(-1000, 1000, n), type=L, mask=rng.random(n) < 0.1)})
    running = [P.window_expr("rn", I, "ROW_NUMBER"), P.window_expr("sv", L, "SUM", [P.col("v")])]
    lead = running + [P.window_expr("ld", L, "LEAD", [P.col("v"), P.lit(1, I), P.lit(None, L)])]
    # running functions only: one output batch per input batch
    got, pulled, total = _stream(_window(t, running), t)
    assert pulled[0] <= 2 and len(pulled) >= 10 and got.num_rows == n
    # LEAD with small partitions: the open partition is held back, the rest goes out
    got_l, pulled_l, _ = _stream(_window(t, lead), t)
    assert pulled_l[0] <= 2 and got_l.num_rows == n
    rows = _cols(got_l, ["p", "o", "v"])
    assert rows == _cols(t, ["p", "o", "v"])
    exp = oracle.window_functions(rows, lambda r: r[0], lambda r: r[1], [("ROW_NUMBER", None, None), ("SUM", lambda r: r[2], None),
                                                                         ("LEAD", lambda r: r[2], (1, lambda r: None))])
    assert _cols(got_l, ["rn", "sv", "ld"]) == exp
    # LEAD without a partition spec: the whole input is one partition, pulled before the first output (as the reference does)
    got_w, pulled_w, total_w = _stream(_window(t, lead, partition=False), t)
    assert pulled_w[0] == total_w and got_w.num_rows == n
    exp_w = oracle.window_functions(rows, lambda r: 0, lambda r: r[1], [("LEAD", lambda r: r[2], (1, lambda r: None))])
    assert [r[0] for r in exp_w] == got_w["ld"].to_pylist()


def test_group_limit_across_batches(prime_batches, monkeypatch):
    keys, rng = _layout(5)
    n = len(keys)
    t = pa.table({"p": pa.array([k[0] for k in keys], type=I), "o": pa.array([k[1] for k in keys], type=L),
                  "s": pa.array([f"s{int(x)}" for x in rng.integers(0, 100, n)])})
    plan = _window(t, [P.window_expr("rk", I, "RANK")], group_limit=2)
    got, pulled, total = _stream(plan, t)
    assert len(pulled) < total                                   # some input batch kept no row, and the stream went on past it
    monkeypatch.delenv("AURON_GPU_CHUNK_ROWS")
    whole = _run(plan, t, chunk=n)
    assert _cols(got, ["p", "o", "s", "rk"]) == _cols(whole, ["p", "o", "s", "rk"])
    exp = [r for r, e in zip(_cols(t, ["p", "o", "s"]), oracle.window_functions(keys, lambda r: r[0], lambda r: r[1], [("RANK", None, None)])) if e[0] <= 2]
    assert _cols(got, ["p", "o", "s"]) == exp


# ---- q51: running SUM per side over aggregated sales, FULL join of the two sides, running MAX of both, filter, top 100
DEC7, DEC17, DEC27 = pa.decimal128(7, 2), pa.decimal128(17, 2), pa.decimal128(27, 2)


def _q51_side(sales_schema, rid, pred, prefix):
    src = P.filter_(P.ffi_reader(sales_schema, rid), [pred])
    keys, names = [P.col("item"), P.col("date")], ["item", "date"]
    partial = P.agg(src, keys, names, [P.agg_expr("SUM", [P.col("price")], DEC17)], ["s"], ["PARTIAL"])
    final = P.agg(partial, keys, names, [P.agg_expr("SUM", [P.lit(None, pa.null())], DEC17)], ["s"], ["FINAL"])
    srt = P.sort(final, [P.sort_expr(P.col("item")), P.sort_expr(P.col("date"))])
    win = P.window(srt, [P.window_expr("cume", DEC27, "SUM", [P.col("s")])], [P.col("item")], [P.sort_expr(P.col("date"))])
    return P.projection(win, [P.col("item"), P.col("date"), P.col("cume")], [f"{prefix}_item", f"{prefix}_date", f"{prefix}_cume"], [I, I, DEC27])


def _q51_plan(sales_schema):
    web = _q51_side(sales_schema, "web", P.binary("Lt", P.col("store"), P.lit(3, I)), "w")
    store = _q51_side(sales_schema, "store", P.binary("GtEq", P.col("store"), P.lit(3, I)), "s")
    js = pa.schema([("w_item", I), ("w_date", I), ("w_cume", DEC27), ("s_item", I), ("s_date", I), ("s_cume", DEC27)])
    j = P.sort_merge_join(js, web, store, [(P.col("w_item"), P.col("s_item")), (P.col("w_date"), P.col("s_date"))], "FULL")
    pick = lambda a, b: P.case([(P.is_not_null(P.col(a)), P.col(a))], P.col(b))
    proj = P.projection(j, [pick("w_item", "s_item"), pick("w_date", "s_date"), P.col("w_cume"), P.col("s_cume")],
                        ["item", "date", "web_sales", "store_sales"], [I, I, DEC27, DEC27])
    srt = P.sort(proj, [P.sort_expr(P.col("item")), P.sort_expr(P.col("date"))])
    win = P.window(srt, [P.window_expr("web_cumulative", DEC27, "MAX", [P.col("web_sales")]), P.window_expr("store_cumulative", DEC27, "MAX", [P.col("store_sales")])],
                   [P.col("item")], [P.sort_expr(P.col("date"))])
    flt = P.filter_(win, [P.binary("Gt", P.col("web_cumulative"), P.col("store_cumulative"))])
    return P.sort(flt, [P.sort_expr(P.col("item")), P.sort_expr(P.col("date"))], limit=100)


def _q51_expected(sales):
    def side(keep):
        acc = {}
        for item, date, store, price in _cols(sales, ["item", "date", "store", "price"]):
            if keep(store):
                cur = acc.get((item, date), "absent")
                acc[(item, date)] = price if cur == "absent" else (cur if price is None else (price if cur is None else cur + price))
        out, run, prev = {}, None, None
        for (item, date) in sorted(acc):
            if item != prev:
                prev, run = item, None
            s = acc[(item, date)]
            if s is not None:
                run = s if run is None else run + s
            out[(item, date)] = run
        return out
    web, store = side(lambda s: s < 3), side(lambda s: s >= 3)
    rows, prev = [], None
    for key in sorted(set(web) | set(store)):
        item, date = key
        if item != prev:
            prev, wmax, smax = item, None, None
        w, s = web.get(key), store.get(key)
        wmax = w if wmax is None else (wmax if w is None else max(wmax, w))
        smax = s if smax is None else (smax if s is None else max(smax, s))
        if wmax is not None and smax is not None and wmax > smax:
            rows.append((item, date, w, s, wmax, smax))
    return rows[:100]


@pytest.mark.parametrize("spill", [False, True])
def test_q51_shape(prime_batches, monkeypatch, spill):
    if spill:
        monkeypatch.setenv("AURON_SORT_SPILL_BYTES", str(64 << 10))   # the sorts emit several ranges into the windows
    rng = np.random.default_rng(51)
    n = 120_000
    sales = pa.table({"item": pa.array(rng.integers(1, 40, n), type=I), "date": pa.array(rng.integers(0, 3_000, n), type=I),
                      "store": pa.array(rng.integers(0, 6, n), type=I),
                      "price": pa.array([D(int(c)).scaleb(-2) for c in rng.integers(0, 20_000, n)], type=DEC7, mask=rng.random(n) < 0.03)})
    td = P.task_definition(_q51_plan(sales.schema))
    got = runtime.run_task(td, {"web": _batches(sales), "store": _batches(sales)})
    exp = _q51_expected(sales)
    assert len(exp) == 100
    names = ["item", "date", "web_sales", "store_sales", "web_cumulative", "store_cumulative"]
    types = [got.schema.field(c).type for c in names]
    assert R.compare("q51", exp, _cols(got, names), types) == []
