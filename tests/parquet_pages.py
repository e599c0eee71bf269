"""A hand-built Parquet file: one INT32 or INT64 column, uncompressed, with exactly the pages a test spells out.

pyarrow's writer chooses its own run layout and never writes some layouts other writers do: a one-entry dictionary whose
indices have bit width 0 (parquet-mr writes it for every column chunk that holds a single value), RLE and bit-packed runs
placed at chosen rows, bit-packed runs of more than 63 groups behind one header.  This writer takes the runs as given.

Runs of the RLE / bit-packed hybrid (definition levels and dictionary indices) are ("rle", count, value) or ("bp", [values]);
a bit-packed run that is not the last of its stream holds a multiple of 8 values, the last one is padded with zeros.
`write` returns the column's values (None for NULL), which the file must read back to through `pq.read_table`.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

# ---- Thrift compact protocol (the subset the footer and page headers need)
_I32, _I64, _BIN, _LIST, _STRUCT, _TRUE, _FALSE = 5, 6, 8, 9, 12, 1, 2


def _varint(n: int) -> bytes:
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _zz(n: int) -> bytes:
    return _varint((n << 1) ^ (n >> 63))


def _struct(fields: list) -> bytes:
    """fields: (id, type, value) in increasing id order; value is an int, bytes, bool, a nested field list, or a list of
    (elem_type, value) for _LIST."""
    out, last = bytearray(), 0
    for fid, ty, v in fields:
        if ty == _TRUE:
            ty = _TRUE if v else _FALSE
        out.append(((fid - last) << 4) | ty)
        last = fid
        if ty in (_I32, _I64):
            out += _zz(v)
        elif ty == _BIN:
            out += _varint(len(v)) + v
        elif ty == _STRUCT:
            out += _struct(v)
        elif ty == _LIST:
            et, items = v
            out.append((len(items) << 4 | et) if len(items) < 15 else (0xF0 | et))
            if len(items) >= 15:
                out += _varint(len(items))
            for it in items:
                out += _zz(it) if et in (_I32, _I64) else (_varint(len(it)) + it if et == _BIN else _struct(it))
    out.append(0)
    return bytes(out)


# ---- RLE / bit-packed hybrid
def hybrid(runs: list, bw: int) -> bytes:
    out = bytearray()
    for k, run in enumerate(runs):
        if run[0] == "rle":
            _, count, value = run
            assert count > 0 and 0 <= value < (1 << bw if bw else 1)
            out += _varint(count << 1) + value.to_bytes((bw + 7) // 8, "little")
        else:
            vals = list(run[1])
            assert vals and (len(vals) % 8 == 0 or k == len(runs) - 1), "only the last bit-packed run may be padded"
            vals += [0] * (-len(vals) % 8)
            out += _varint((len(vals) // 8) << 1 | 1)
            acc = 0
            for i, v in enumerate(vals):
                assert 0 <= v < (1 << bw if bw else 1)
                acc |= v << (i * bw)
            out += acc.to_bytes(len(vals) * bw // 8, "little")
    return bytes(out)


def expand(runs: list) -> list:
    out = []
    for run in runs:
        out += [run[2]] * run[1] if run[0] == "rle" else list(run[1])
    return out


@dataclass
class Page:
    n: int                                        # rows of the page
    def_runs: list | None = None                  # OPTIONAL columns: definition levels (bit width 1)
    idx_runs: list | None = None                  # dictionary pages: indices of the non-null values ...
    bw: int = 0                                   # ... at this bit width
    plain: list = field(default_factory=list)     # PLAIN pages: the non-null values
    v2: bool = False


def write(path: str, physical: str, required: bool, pages: list, dictionary: list | None = None, name: str = "c", stats: bool = False) -> list:
    """stats: write the chunk's min / max / null count (Statistics fields 5, 6, 3)."""
    ptype, fmt = {"INT32": (1, "<i"), "INT64": (2, "<q")}[physical]
    body, values, encodings = bytearray(), [], set()
    dict_off = None
    if dictionary is not None:
        raw = b"".join(struct.pack(fmt, v) for v in dictionary)
        hdr = _struct([(1, _I32, 2), (2, _I32, len(raw)), (3, _I32, len(raw)), (7, _STRUCT, [(1, _I32, len(dictionary)), (2, _I32, 0)])])
        dict_off = 4
        body += hdr + raw
        encodings.add(0)
    data_off = 4 + len(body)
    for pg in pages:
        levels = [1] * pg.n if required else expand(pg.def_runs)[:pg.n]
        assert len(levels) == pg.n
        nn = sum(levels)
        if pg.idx_runs is not None:
            idx = expand(pg.idx_runs)[:nn]
            assert len(idx) == nn
            vals = iter(dictionary[i] for i in idx)
            vsec, enc = bytes([pg.bw]) + hybrid(pg.idx_runs, pg.bw), 8
        else:
            assert len(pg.plain) == nn
            vals = iter(pg.plain)
            vsec, enc = b"".join(struct.pack(fmt, v) for v in pg.plain), 0
        encodings.add(enc)
        values += [next(vals) if lv else None for lv in levels]
        dsec = b"" if required else hybrid(pg.def_runs, 1)
        if pg.v2:
            payload = dsec + vsec
            hdr = _struct([(1, _I32, 3), (2, _I32, len(payload)), (3, _I32, len(payload)),
                           (8, _STRUCT, [(1, _I32, pg.n), (2, _I32, pg.n - nn), (3, _I32, pg.n), (4, _I32, enc), (5, _I32, len(dsec)), (6, _I32, 0),
                                         (7, _TRUE, False)])])
        else:
            payload = (struct.pack("<I", len(dsec)) + dsec if not required else b"") + vsec
            hdr = _struct([(1, _I32, 0), (2, _I32, len(payload)), (3, _I32, len(payload)),
                           (5, _STRUCT, [(1, _I32, pg.n), (2, _I32, enc), (3, _I32, 3), (4, _I32, 3)])])
        body += hdr + payload
    rows = sum(pg.n for pg in pages)
    meta = [(1, _I32, ptype), (2, _LIST, (_I32, sorted(encodings | {3}))), (3, _LIST, (_BIN, [name.encode()])), (4, _I32, 0), (5, _I64, rows),
            (6, _I64, len(body)), (7, _I64, len(body)), (9, _I64, data_off)]
    if dict_off is not None:
        meta.append((11, _I64, dict_off))
    nonnull = [v for v in values if v is not None]
    if stats:
        st = [(3, _I64, len(values) - len(nonnull))]
        if nonnull:
            st += [(5, _BIN, struct.pack(fmt, max(nonnull))), (6, _BIN, struct.pack(fmt, min(nonnull)))]
        meta.append((12, _STRUCT, st))
    footer = _struct([
        (1, _I32, 2),
        (2, _LIST, (_STRUCT, [[(4, _BIN, b"schema"), (5, _I32, 1)], [(1, _I32, ptype), (3, _I32, 0 if required else 1), (4, _BIN, name.encode())]])),
        (3, _I64, rows),
        (4, _LIST, (_STRUCT, [[(1, _LIST, (_STRUCT, [[(2, _I64, 4), (3, _STRUCT, meta)]])), (2, _I64, len(body)), (3, _I64, rows)]])),
    ])
    with open(path, "wb") as f:
        f.write(b"PAR1" + bytes(body) + footer + struct.pack("<I", len(footer)) + b"PAR1")
    return values


def layouts() -> list:
    """The hand-built layouts the suite scans: (id, physical, required, pages, dictionary)."""
    P = Page
    edge32 = [-2**31, 2**31 - 1, 0, 1, -1]
    out = [
        # parquet-mr's single-value chunk: a one-entry dictionary, indices of bit width 0
        ("bw0_required_v1", "INT32", True, [P(n=1025, idx_runs=[("rle", 1025, 0)], bw=0)], [123456]),
        ("bw0_optional_v2", "INT64", False, [P(n=1060, def_runs=[("rle", 31, 1), ("rle", 2, 0), ("rle", 990, 0), ("rle", 37, 1)], idx_runs=[("rle", 68, 0)], bw=0,
                                              v2=True)], [-2**63]),
        ("bw0_bitpacked_v1", "INT32", False, [P(n=77, def_runs=[("bp", [1, 0, 1, 1, 0, 1, 1, 1] * 9 + [1, 1, 0, 1, 1])], idx_runs=[("bp", [0] * 64)], bw=0)],
         [-7]),
    ]
    # RLE runs of 1, 7, 8, 31-33 and 1023-1025 rows, alternating entries, one page per format
    lens = [1, 7, 8, 31, 32, 33, 1023, 1024, 1025]
    runs = [("rle", k, i % 5) for i, k in enumerate(lens)]
    for v2 in (False, True):
        out.append((f"rle_runs_{'v2' if v2 else 'v1'}", "INT32", True, [P(n=sum(lens), idx_runs=runs, bw=3, v2=v2)], edge32))
    # bit-packed runs of 1 group, 63 groups and 100 groups behind one header; the page ends inside a padded group
    bp = [("bp", [i % 17 for i in range(8)]), ("bp", [(3 * i) % 17 for i in range(63 * 8)]), ("rle", 9, 16), ("bp", [(5 * i + 1) % 17 for i in range(797)])]
    n_bp = 8 + 63 * 8 + 9 + 797
    out.append(("bitpacked_groups_i64", "INT64", True, [P(n=n_bp, idx_runs=bp, bw=5)], [(-1) ** i * (2**62 + i) for i in range(17)]))
    out.append(("bitpacked_groups_bw32", "INT32", True, [P(n=n_bp, idx_runs=bp, bw=32, v2=True)], list(range(-8, 9))))
    # NULL runs one row either side of multiples of 32 and 1024, over three pages (v1, v2, v1) with a dictionary and PLAIN pages
    d1 = [("rle", 31, 1), ("rle", 2, 0), ("rle", 990, 1), ("rle", 2, 0), ("bp", [1, 0, 1, 1, 0, 0, 1, 0] * 4), ("rle", 1, 1)]
    n1 = 31 + 2 + 990 + 2 + 32 + 1
    nn1 = 31 + 990 + 16 + 1
    out.append(("null_runs_pages", "INT32", False, [
        P(n=n1, def_runs=d1, idx_runs=[("bp", [i % 6 for i in range(nn1 - nn1 % 8)]), ("rle", nn1 % 8, 5)], bw=3),
        P(n=7, def_runs=[("rle", 7, 0)], idx_runs=[], bw=1, v2=True),
        P(n=1025, def_runs=[("rle", 1023, 1), ("rle", 1, 0), ("rle", 1, 1)], plain=[(i * 7919) % 2**31 - 2**30 for i in range(1024)]),
    ], edge32 + [5]))
    return out
