"""Plain-Python, bytes-level reference of the VM's string functions: lpad, rpad, replace, translate, reverse, initcap, ascii,
bit_length, find_in_set and trim with a character set.

Values are bytes (utf8 as its encoded bytes), integers as Python ints, NULL as None; a NULL argument gives NULL.  A character
is a lead byte and the continuation bytes it announces, cut at the end of the value, which is what CharacterLength and Substr
count.  Only plain Python is used -- no engine, no numpy, no Arrow.

Semantics (Spark's, which the device follows):
  * lpad / rpad (UTF8String.lpad / rpad): n <= 0 -> ""; n below the character count truncates to the first n characters; an
    empty pad returns s; otherwise the pad characters repeat, cycling, cut to n characters in all, before (lpad) or after s
  * replace (UTF8String.replace): non-overlapping matches found left to right; an empty search returns s unchanged
  * translate (StringTranslate): the k-th character of `from` becomes the k-th of `to`, or is deleted when `to` has no k-th;
    a character repeated in `from` keeps its first position, and later duplicates still use up their position in `to`
  * reverse: the characters in reverse order
  * initcap (spark_initcap.rs:40-66 for ASCII): an ASCII letter or digit first or after ' ' is upper-cased, every other ASCII
    letter lower-cased; other bytes are copied
  * ascii: the code point of the first character, 0 for ""
  * bit_length: 8 x the byte length
  * find_in_set (UTF8String.findInSet): the 1-based index of s among the comma-separated pieces of the list; 0 when s holds
    a comma or is not there
  * btrim / ltrim / rtrim with a set: the characters of the set removed from the chosen end(s)
"""
from __future__ import annotations


def char_len(b: int) -> int:
    return 1 if b < 0x80 else 2 if b >> 5 == 6 else 3 if b >> 4 == 14 else 4 if b >> 3 == 30 else 1


def chars(s: bytes) -> list[bytes]:
    try:   # well-formed UTF-8 splits the same way; the codec does it faster
        return [c.encode() for c in s.decode()]
    except UnicodeDecodeError:
        pass
    out, i = [], 0
    while i < len(s):
        k = min(char_len(s[i]), len(s) - i)
        out.append(s[i:i + k])
        i += k
    return out


def _pad(s, n, pad, left):
    if s is None or n is None or pad is None:
        return None
    if n <= 0:
        return b""
    cs = chars(s)
    if len(cs) >= n or not pad:
        return b"".join(cs[:n])
    pc = chars(pad)
    k = n - len(cs)
    fill = pad * (k // len(pc)) + b"".join(pc[:k % len(pc)])
    return fill + s if left else s + fill


def lpad(s, n, pad):
    return _pad(s, n, pad, True)


def rpad(s, n, pad):
    return _pad(s, n, pad, False)


def pad_len(s: bytes, n: int, pad: bytes) -> int:
    """the byte length lpad / rpad would produce, without building the value (n may be as large as 2^63 - 1)"""
    if n <= 0:
        return 0
    cs = chars(s)
    if len(cs) >= n or not pad:
        return len(b"".join(cs[:n]))
    pc = chars(pad)
    k = n - len(cs)
    return len(s) + len(pad) * (k // len(pc)) + len(b"".join(pc[:k % len(pc)]))


def replace(s, search, rep):
    if s is None or search is None or rep is None:
        return None
    if not search:
        return s
    return s.replace(search, rep)   # bytes.replace: non-overlapping matches, left to right


def translate(s, frm, to):
    if s is None or frm is None or to is None:
        return None
    fc, tc = chars(frm), chars(to)
    table = {}
    for k, c in enumerate(fc):
        table.setdefault(c, tc[k] if k < len(tc) else b"")
    return b"".join(table.get(c, c) for c in chars(s))


def reverse(s):
    return None if s is None else b"".join(reversed(chars(s)))


def initcap(s):
    if s is None:
        return None
    out, after_space = bytearray(), True
    for c in s:
        if after_space and 0x61 <= c <= 0x7a:
            c -= 32
        elif not after_space and 0x41 <= c <= 0x5a:
            c += 32
        out.append(c)
        after_space = c == 0x20
    return bytes(out)


def ascii_(s):
    if s is None:
        return None
    if not s:
        return 0
    c = chars(s)[0]
    if len(c) == 1:
        return c[0]
    v = c[0] & (0x7f >> len(c))
    for b in c[1:]:
        v = (v << 6) | (b & 0x3f)
    return v


def bit_length(s):
    return None if s is None else 8 * len(s)


def find_in_set(s, lst):
    if s is None or lst is None:
        return None
    if b"," in s:
        return 0
    for k, piece in enumerate(lst.split(b","), 1):
        if piece == s:
            return k
    return 0


def trim(s, chars_set, sides: str = "both"):
    """sides: 'both' (Trim / Btrim), 'left' (Ltrim) or 'right' (Rtrim)"""
    if s is None or chars_set is None:
        return None
    cs, st = chars(s), set(chars(chars_set))
    b, e = 0, len(cs)
    if sides in ("both", "left"):
        while b < e and cs[b] in st:
            b += 1
    if sides in ("both", "right"):
        while e > b and cs[e - 1] in st:
            e -= 1
    return b"".join(cs[b:e])


def upper(s):   # the VM's ASCII-only upper / lower
    return None if s is None else bytes(c - 32 if 0x61 <= c <= 0x7a else c for c in s)


def lower(s):
    return None if s is None else bytes(c + 32 if 0x41 <= c <= 0x5a else c for c in s)
