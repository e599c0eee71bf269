"""Hand-built Parquet files with one top-level LIST column in a chosen schema form, uncompressed, with the level pages a test spells out.

pyarrow writes only the standard 3-level form and cuts its pages at row boundaries.  Older writers use the 2-level forms and the
bare repeated field of parquet-format's LogicalTypes.md ("Backward-compatibility rules"), and a v1 page may start inside a row
(its first repetition level is 1).  This writer takes the schema form and the page cuts as given; `pq.read_table` reads the files back.

`write(path, form, rows, cuts=...)`: rows are None (a NULL list) or lists of ints / None; `cuts` are the slot positions where a new page
starts.  Forms that hold structs are written without row groups: only their schema is looked at.
"""
from __future__ import annotations

import struct

from parquet_pages import _BIN, _I32, _I64, _LIST, _STRUCT, _TRUE, _struct, hybrid

REQ, OPT, REP = 0, 1, 2
LIST, MAP = 3, 1   # converted types

# form -> (schema elements below the root as (name, repetition, num_children, converted_type, physical type or None), list_def, elem_def,
#          max_def, readable).  `{n}` is the column's name; `{e}` the element's repetition.
FORMS = {
    "standard":          ([("{n}", OPT, 1, LIST, None), ("list", REP, 1, None, None), ("element", "{e}", 0, None, "P")], True),
    "pyarrow_item":      ([("{n}", OPT, 1, LIST, None), ("list", REP, 1, None, None), ("item", "{e}", 0, None, "P")], True),
    "spark_bag_array":   ([("{n}", OPT, 1, LIST, None), ("bag", REP, 1, None, None), ("array", "{e}", 0, None, "P")], True),
    "hive_array_element": ([("{n}", OPT, 1, LIST, None), ("bag", REP, 1, None, None), ("array_element", "{e}", 0, None, "P")], True),
    "required_standard": ([("{n}", REQ, 1, LIST, None), ("list", REP, 1, None, None), ("element", "{e}", 0, None, "P")], True),
    "two_level_primitive": ([("{n}", OPT, 1, LIST, None), ("array", REP, 0, None, "P")], True),
    "bare_repeated":     ([("{n}", REP, 0, None, "P")], True),
    "array_group":       ([("{n}", OPT, 1, LIST, None), ("array", REP, 1, None, None), ("x", REQ, 0, None, "P")], False),
    "tuple_group":       ([("{n}", OPT, 1, LIST, None), ("{n}_tuple", REP, 1, None, None), ("x", REQ, 0, None, "P")], False),
    "multi_field_group": ([("{n}", OPT, 1, LIST, None), ("rec", REP, 2, None, None), ("x", REQ, 0, None, "P"), ("y", OPT, 0, None, "P")], False),
    "list_of_lists":     ([("{n}", OPT, 1, LIST, None), ("list", REP, 1, None, None), ("element", OPT, 1, LIST, None), ("list", REP, 1, None, None),
                           ("element", OPT, 0, None, "P")], False),
    "map":               ([("{n}", OPT, 1, MAP, None), ("key_value", REP, 2, None, None), ("key", REQ, 0, None, "P"), ("value", OPT, 0, None, "P")], False),
    "struct":            ([("{n}", OPT, 2, None, None), ("a", OPT, 0, None, "P"), ("b", REQ, 0, None, "P")], False),
    "repeated_group":    ([("{n}", REP, 1, None, None), ("x", OPT, 0, None, "P")], False),
}
# the shape the engine's schema walk must give each form
SHAPES = {"standard": "list", "pyarrow_item": "list", "spark_bag_array": "list", "hive_array_element": "list", "required_standard": "list",
          "two_level_primitive": "list", "bare_repeated": "list", "array_group": "list of structs", "tuple_group": "list of structs",
          "multi_field_group": "list of structs", "list_of_lists": "list of lists", "map": "map", "struct": "struct", "repeated_group": "list of structs"}


def levels_of(form: str, elem_required: bool):
    """(list_def, elem_def, max_def) of a readable form"""
    elems, _ = FORMS[form]
    top = elems[0][1]
    list_def = 1 if top == OPT else 0
    elem_def = list_def + 1
    three_level = len(elems) == 3
    return list_def, elem_def, elem_def + (1 if three_level and not elem_required else 0)


def _schema(form, name, ptype, elem_required):
    elems, _ = FORMS[form]
    out = [[(4, _BIN, b"schema"), (5, _I32, 1)]]
    for nm, rep, nch, conv, phys in elems:
        rep = (REQ if elem_required else OPT) if rep == "{e}" else rep
        f = []
        if phys:
            f.append((1, _I32, ptype))
        f += [(3, _I32, rep), (4, _BIN, nm.replace("{n}", name).encode())]
        if nch:
            f.append((5, _I32, nch))
        if conv is not None:
            f.append((6, _I32, conv))
        out.append(f)
    return out


def _encode_levels(levels: list, bw: int) -> bytes:
    """RLE runs for stretches of 8+ equal levels, bit-packed groups of 8 otherwise (the last run padded)"""
    runs, i, n = [], 0, len(levels)
    while i < n:
        j = i
        while j < n and levels[j] == levels[i]:
            j += 1
        if j - i >= 8:
            runs.append(("rle", j - i, levels[i]))
            i = j
        else:
            runs.append(("bp", levels[i:i + 8]))
            i += 8
    return hybrid(runs, bw)


def slots_of(rows: list, list_def: int, elem_def: int, max_def: int):
    """[(rep, def, value or None)] of the rows"""
    out = []
    for r in rows:
        if r is None:
            assert list_def > 0, "a required list has no NULL rows"
            out.append((0, list_def - 1, None))
        elif not r:
            out.append((0, list_def, None))
        else:
            for k, v in enumerate(r):
                assert v is not None or max_def > elem_def, "a required element has no NULLs"
                out.append((0 if k == 0 else 1, max_def if v is not None else elem_def, v))
    return out


def write(path: str, form: str, rows: list, cuts: tuple = (), physical: str = "INT32", elem_required: bool = False, v2: bool = False, name: str = "l"):
    ptype, fmt = {"INT32": (1, "<i"), "INT64": (2, "<q")}[physical]
    elems, readable = FORMS[form]
    schema = _schema(form, name, ptype, elem_required)
    leaf_path = [e[0].replace("{n}", name).encode() for e in elems]
    if not readable:
        footer = _struct([(1, _I32, 2), (2, _LIST, (_STRUCT, schema)), (3, _I64, 0), (4, _LIST, (_STRUCT, []))])
        with open(path, "wb") as f:
            f.write(b"PAR1" + footer + struct.pack("<I", len(footer)) + b"PAR1")
        return
    list_def, elem_def, max_def = levels_of(form, elem_required)
    slots = slots_of(rows, list_def, elem_def, max_def)
    bounds = [0] + sorted(c for c in cuts if 0 < c < len(slots)) + [len(slots)]
    dbw = max_def.bit_length()
    body = bytearray()
    for a, b in zip(bounds, bounds[1:]):
        pg = slots[a:b]
        rsec = _encode_levels([s[0] for s in pg], 1)
        dsec = _encode_levels([s[1] for s in pg], dbw)
        vals = [s[2] for s in pg if s[1] == max_def]
        vsec = b"".join(struct.pack(fmt, v) for v in vals)
        if v2:
            payload = rsec + dsec + vsec
            hdr = _struct([(1, _I32, 3), (2, _I32, len(payload)), (3, _I32, len(payload)),
                           (8, _STRUCT, [(1, _I32, len(pg)), (2, _I32, len(pg) - len(vals)), (3, _I32, sum(s[0] == 0 for s in pg)), (4, _I32, 0),
                                         (5, _I32, len(dsec)), (6, _I32, len(rsec)), (7, _TRUE, False)])])
        else:
            payload = struct.pack("<I", len(rsec)) + rsec + struct.pack("<I", len(dsec)) + dsec + vsec
            hdr = _struct([(1, _I32, 0), (2, _I32, len(payload)), (3, _I32, len(payload)),
                           (5, _STRUCT, [(1, _I32, len(pg)), (2, _I32, 0), (3, _I32, 3), (4, _I32, 3)])])
        body += hdr + payload
    meta = [(1, _I32, ptype), (2, _LIST, (_I32, [0, 3])), (3, _LIST, (_BIN, leaf_path)), (4, _I32, 0), (5, _I64, len(slots)),
            (6, _I64, len(body)), (7, _I64, len(body)), (9, _I64, 4)]
    footer = _struct([
        (1, _I32, 2),
        (2, _LIST, (_STRUCT, schema)),
        (3, _I64, len(rows)),
        (4, _LIST, (_STRUCT, [[(1, _LIST, (_STRUCT, [[(2, _I64, 4), (3, _STRUCT, meta)]])), (2, _I64, len(body)), (3, _I64, len(rows))]])),
    ])
    with open(path, "wb") as f:
        f.write(b"PAR1" + bytes(body) + footer + struct.pack("<I", len(footer)) + b"PAR1")
