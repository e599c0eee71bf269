"""Plain-Python restatement of the reference's explode / posexplode and of the two list constructors the engine computes, as the tests
compare against them (paths relative to native-engine/):

  * explode / posexplode (datafusion-ext-plans/src/generate_exec.rs:191-310, generate/explode.rs): rows come out in input order and
    each row's elements in list order; a NULL element gives a row with a NULL value; a NULL or empty list gives no row, or with
    `outer` exactly one row whose generated columns (the position included) are NULL.
  * Spark_StringSplit (datafusion-ext-functions/src/spark_strings.rs:93-115): Rust's str::split by a literal pattern -- leftmost
    non-overlapping matches, "" gives [""], a trailing separator gives a trailing "", a NULL string gives a NULL list.
  * Spark_MakeArray (datafusion-ext-functions/src/spark_make_array.rs): one list of the arguments per row; elements may be NULL,
    the list never is.

Lists are Python lists (None = NULL list); rows are tuples.
"""
from __future__ import annotations


def string_split(s: str | bytes | None, pattern: str | bytes) -> list | None:
    """str::split: the pieces between the leftmost non-overlapping matches of `pattern` (non-empty)"""
    if s is None:
        return None
    assert len(pattern) > 0
    out, start = [], 0
    while True:
        i = s.find(pattern, start)
        if i < 0:
            out.append(s[start:])
            return out
        out.append(s[start:i])
        start = i + len(pattern)


def make_array(*args: list) -> list[list]:
    """array(a1, .., aN) over columns of one length (a scalar argument is a column of that value)"""
    return [list(vals) for vals in zip(*args)]


def explode(rows: list[tuple], lists: list[list | None], pos: bool = False, outer: bool = False) -> list[tuple]:
    """the output rows of GenerateExec: each input row's required values followed by [position,] element"""
    out = []
    for req, lst in zip(rows, lists):
        if not lst:   # NULL or empty
            if outer:
                out.append(tuple(req) + ((None, None) if pos else (None,)))
            continue
        for k, v in enumerate(lst):
            out.append(tuple(req) + ((k, v) if pos else (v,)))
    return out


def list_offsets(lists: list[list | None]) -> list[int]:
    """Arrow offsets of a list column (a NULL list covers no elements)"""
    offs = [0]
    for lst in lists:
        offs.append(offs[-1] + (len(lst) if lst is not None else 0))
    return offs
