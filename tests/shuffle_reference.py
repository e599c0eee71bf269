"""Plain-Python references for the shuffle byte format: the compacted batch layout of batch_serde.rs (write_batch / read_batch,
batch_serde.rs:68-101,273-346 and the bits / bytes writers), the LZ4 frame format and the LZ4 block format.

Values are in key_reference's canonical form: ints, dates, timestamps and unscaled decimals as Python ints, floats as their IEEE
bits, bool as bool, utf8 / binary as bytes, NULL as None.  Type names are key_reference.TYPES plus "null".  Only Python ints,
struct and bytes are used here -- no engine, no Arrow, no compression library."""
from __future__ import annotations

import struct

import key_reference as R

FIXED_WIDTH = {"int8": 1, "int16": 2, "int32": 4, "int64": 8, "float32": 4, "float64": 8, "date32": 4, "date64": 8,
               **{t: 8 for t in R.TIMESTAMPS}, **{t: 16 for t in R.DECIMALS}}
LZ4_MAGIC = 0x184D2204
LZ4_BLOCK_MAX = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}


def _check(cond, msg):
    if not cond:
        raise AssertionError(msg)


# -------------------------------------------------------------------------------------------- varints and bit sections
def write_len(v: int) -> bytes:
    """io/mod.rs write_len: 7 bits per byte, low bits first, high bit = more bytes follow"""
    out = bytearray()
    while v >= 128:
        out.append(128 + v % 128)
        v //= 128
    out.append(v)
    return bytes(out)


def read_len(buf, pos: int):
    v, shift = 0, 0
    while True:
        _check(pos < len(buf) and shift < 64, "truncated varint")
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << shift
        if not b & 0x80:
            return v, pos
        shift += 7


def pack_bits(flags) -> bytes:
    """write_bits_buffer: bit i of the section = flags[i], re-based to bit 0, padding bits zero"""
    out = bytearray((len(flags) + 7) // 8)
    for i, f in enumerate(flags):
        if f:
            out[i >> 3] |= 1 << (i & 7)
    return bytes(out)


def unpack_bits(sec: bytes, n: int) -> list[bool]:
    _check(len(sec) == (n + 7) // 8, "bit section length")
    _check(n % 8 == 0 or sec[-1] >> (n % 8) == 0, "padding bits of a bit section are not zero")
    return [bool(sec[i >> 3] >> (i & 7) & 1) for i in range(n)]


def _signed(t: str) -> bool:
    return t not in R.FLOATS


# -------------------------------------------------------------------------------------------- batch layout
def write_batch(columns, has_nulls) -> bytes:
    """write_batch: varint num_rows | column*.  columns = [(type, values)] of equal length; has_nulls[c] = the column's flag
    (1: a validity section follows, also when no value is NULL; 0 is only possible without NULLs).  NULL slots are written
    with zero values, an empty string and a clear bool bit."""
    n = len(columns[0][1]) if columns else 0
    out = bytearray(write_len(n))
    for (t, vals), hn in zip(columns, has_nulls):
        _check(len(vals) == n, "ragged batch")
        if t == "null":                                  # DataType::Null writes nothing
            continue
        _check(hn or all(v is not None for v in vals), f"{t}: NULL value in a column written without a validity section")
        out += write_len(1 if hn else 0)
        if hn:
            out += pack_bits([v is not None for v in vals])
        if t == "bool":
            out += pack_bits([bool(v) for v in vals])
        elif t in ("utf8", "binary"):
            data = [b"" if v is None else v for v in vals]
            lens = b"".join(struct.pack("<i", len(v)) for v in data)
            out += b"".join(lens[k::4] for k in range(4))          # four transposed i32 planes
            out += b"".join(data)
        else:
            w = FIXED_WIDTH[t]
            raw = b"".join((0 if v is None else v).to_bytes(w, "little", signed=_signed(t)) for v in vals)
            out += raw if w == 1 else b"".join(raw[k::w] for k in range(w))   # byte planes for widths >= 2
    return bytes(out)


def _untranspose(sec: bytes, w: int, n: int) -> bytes:
    _check(len(sec) == w * n, "truncated byte planes")
    raw = bytearray(w * n)
    for k in range(w):
        raw[k::w] = sec[k * n:(k + 1) * n]
    return bytes(raw)


def read_sections(payload: bytes, schema) -> list[dict]:
    """read_batch over a whole payload (a sequence of batches).  schema = list of type names.  Per batch: n, start / end byte
    of the batch in the payload, and per column has_nulls, the values (None for NULL) and the offset of its value section
    (the first byte plane, the bool bits or the length planes).  Asserts that the payload ends with a whole batch."""
    batches, pos = [], 0
    while pos < len(payload):
        start = pos
        n, pos = read_len(payload, pos)
        cols, hns, voffs = [], [], []
        for t in schema:
            if t == "null":
                cols.append([None] * n)
                hns.append(None)
                voffs.append(None)
                continue
            hn, pos = read_len(payload, pos)
            _check(hn in (0, 1), f"has_nulls = {hn}")
            valid = [True] * n
            if hn:
                valid = unpack_bits(payload[pos:pos + (n + 7) // 8], n)
                pos += (n + 7) // 8
            voffs.append(pos)
            if t == "bool":
                vals = unpack_bits(payload[pos:pos + (n + 7) // 8], n)
                pos += (n + 7) // 8
            elif t in ("utf8", "binary"):
                lens = struct.unpack(f"<{n}i", _untranspose(payload[pos:pos + 4 * n], 4, n))
                pos += 4 * n
                vals = []
                for ln in lens:
                    _check(ln >= 0, "negative string length")
                    vals.append(payload[pos:pos + ln])
                    pos += ln
            else:
                w = FIXED_WIDTH[t]
                sec = payload[pos:pos + w * n]
                pos += w * n
                raw = sec if w == 1 else _untranspose(sec, w, n)
                vals = [int.from_bytes(raw[i * w:(i + 1) * w], "little", signed=_signed(t)) for i in range(n)]
            _check(pos <= len(payload), "batch overruns the payload")
            cols.append([v if ok else None for v, ok in zip(vals, valid)])
            hns.append(hn)
        batches.append({"n": n, "start": start, "end": pos, "cols": cols, "has_nulls": hns, "values_off": voffs})
    return batches


# -------------------------------------------------------------------------------------------- xxHash32
_P1, _P2, _P3, _P4, _P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
_M32 = 0xFFFFFFFF


def _rotl(x: int, r: int) -> int:
    return ((x << r) | (x >> (32 - r))) & _M32


def xxh32(data: bytes, seed: int = 0) -> int:
    n, p = len(data), 0
    if n >= 16:
        v = [(seed + _P1 + _P2) & _M32, (seed + _P2) & _M32, seed & _M32, (seed - _P1) & _M32]
        while p + 16 <= n:
            for i in range(4):
                lane = int.from_bytes(data[p:p + 4], "little")
                v[i] = (_rotl((v[i] + lane * _P2) & _M32, 13) * _P1) & _M32
                p += 4
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M32
    else:
        h = (seed + _P5) & _M32
    h = (h + n) & _M32
    while p + 4 <= n:
        h = (_rotl((h + int.from_bytes(data[p:p + 4], "little") * _P3) & _M32, 17) * _P4) & _M32
        p += 4
    while p < n:
        h = (_rotl((h + data[p] * _P5) & _M32, 11) * _P1) & _M32
        p += 1
    h ^= h >> 15
    h = (h * _P2) & _M32
    h ^= h >> 13
    h = (h * _P3) & _M32
    return h ^ (h >> 16)


def header_checksum(descriptor: bytes) -> int:
    """HC of an LZ4 frame header: the second byte of xxh32 over the frame descriptor (FLG .. optional fields)"""
    return (xxh32(descriptor) >> 8) & 0xFF


# -------------------------------------------------------------------------------------------- LZ4 frames
def split_streams(segment: bytes) -> list[bytes]:
    """a shuffle segment = (u32_le len | codec stream)*: the streams, each with its length word, nothing left over"""
    out, pos = [], 0
    while pos < len(segment):
        _check(pos + 4 <= len(segment), "truncated stream length")
        (ln,) = struct.unpack_from("<I", segment, pos)
        _check(ln > 0 and pos + 4 + ln <= len(segment), "stream overruns its segment")
        out.append(segment[pos:pos + 4 + ln])
        pos += 4 + ln
    return out


def lz4_frame_blocks(stream: bytes) -> dict:
    """Walks one codec stream: u32 length, magic, FLG / BD / HC, each block's size word (high bit = stored) and data
    (+ block checksum), the end mark (+ content checksum).  Asserts that the length word covers exactly the frame."""
    (ln,) = struct.unpack_from("<I", stream, 0)
    _check(ln == len(stream) - 4, f"stream length word {ln} != {len(stream) - 4}")
    f = stream[4:]
    _check(len(f) >= 7 and struct.unpack_from("<I", f, 0)[0] == LZ4_MAGIC, "not an LZ4 frame")
    flg, bd = f[4], f[5]
    _check(flg >> 6 == 1, "frame version")
    _check(flg & 0x02 == 0 and bd & 0x8F == 0, "reserved header bits set")
    _check((bd >> 4) & 7 in LZ4_BLOCK_MAX, "block maximum size")
    pos = 6 + (8 if flg & 0x08 else 0) + (4 if flg & 0x01 else 0)
    _check(pos < len(f), "truncated frame header")
    hc = f[pos]
    _check(hc == header_checksum(f[4:pos]), f"header checksum {hc:#04x} != {header_checksum(f[4:pos]):#04x}")
    pos += 1
    info = {"flg": flg, "bd": bd, "hc": hc, "linked": not flg & 0x20, "block_max": LZ4_BLOCK_MAX[(bd >> 4) & 7], "blocks": [],
            "content_size": int.from_bytes(f[6:14], "little") if flg & 0x08 else None, "content_checksum": None}
    while True:
        _check(pos + 4 <= len(f), "truncated block size word")
        (w,) = struct.unpack_from("<I", f, pos)
        pos += 4
        if w == 0:
            break
        size = w & 0x7FFFFFFF
        _check(size <= info["block_max"], f"block of {size} bytes over the block maximum")
        _check(pos + size <= len(f), "block overruns the frame")
        data = f[pos:pos + size]
        pos += size
        if flg & 0x10:
            _check(struct.unpack_from("<I", f, pos)[0] == xxh32(data), "block checksum")
            pos += 4
        info["blocks"].append((bool(w >> 31), data))
    if flg & 0x04:
        info["content_checksum"] = struct.unpack_from("<I", f, pos)[0]
        pos += 4
    _check(pos == len(f), f"{len(f) - pos} bytes after the end mark")
    return info


def lz4_frame_decode(info: dict, stats: dict | None = None) -> bytes:
    """The content of a walked frame: stored blocks as they are, compressed blocks through lz4_block_decode (linked blocks see
    the last 64 KB of the previous output), the content size and checksum checked when the frame carries them."""
    out = bytearray()
    for stored, data in info["blocks"]:
        if stored:
            out += data
            continue
        hist = bytes(out[-65536:]) if info["linked"] else b""
        blk, _ = lz4_block_decode(data, history=hist, stats=stats, max_len=info["block_max"])
        out += blk
    if info["content_size"] is not None:
        _check(len(out) == info["content_size"], "content size")
    if info["content_checksum"] is not None:
        _check(xxh32(bytes(out)) == info["content_checksum"], "content checksum")
    return bytes(out)


def lz4_frame(blocks) -> bytes:
    """An LZ4 frame with independent 64 KB blocks and no checksums (what lz4_flex's FrameEncoder writes), from
    [(raw bytes, compressed block)]: a block is stored raw when compressing did not make it smaller.  No length word."""
    descriptor = bytes([0x60, 0x40])
    out = bytearray(struct.pack("<I", LZ4_MAGIC) + descriptor + bytes([header_checksum(descriptor)]))
    for raw, comp in blocks:
        if len(comp) >= len(raw):
            out += struct.pack("<I", len(raw) | 0x80000000) + raw
        else:
            out += struct.pack("<I", len(comp)) + comp
    return bytes(out + b"\0\0\0\0")


# -------------------------------------------------------------------------------------------- LZ4 blocks
MINMATCH, MFLIMIT, LASTLITERALS = 4, 12, 5


def new_stats() -> dict:
    return {"blocks": 0, "matches": 0, "min_offset": None, "max_offset": 0, "overlapping": 0, "long_literals": 0, "max_literal": 0,
            "literal_lengths": set(), "match_lengths": set(), "small_offset_runs": set(), "max_overlap_len_off_ge4": 0,
            "short_overlaps": 0, "far_offsets": 0}


def _ext(block: bytes, ip: int, v: int):
    if v == 15:
        while True:
            _check(ip < len(block), "truncated length extension")
            x = block[ip]
            ip += 1
            v += x
            if x != 255:
                break
    return v, ip


def lz4_block_decode(block: bytes, expected_len: int | None = None, history: bytes = b"", stats: dict | None = None,
                     max_len: int = 1 << 30):
    """Strict LZ4 block decoder -> (bytes, stats).  Asserts the exact output length (when given), 1 <= offset <= bytes available
    (this block's output plus `history`, the previous output of a linked frame), and the end-of-block rules: the last sequence is
    literals only, and when the block has a match, the last 5 bytes are literals and the last match starts at least 12 bytes
    before the end.  Statistics (merged into `stats` when given): offsets, overlapping matches (offset < length), literal runs
    over 256 bytes, (offset, output position & 3) of runs with offset <= 3 and length >= 64, overlapping runs with offset >= 4."""
    st = stats if stats is not None else new_stats()
    st["blocks"] += 1
    out = bytearray(history)
    base = len(history)
    ip, last_match_start, last_seq_has_match = 0, None, False
    _check(len(block) > 0, "empty block")
    while True:
        _check(ip < len(block), "truncated block: missing token")
        token = block[ip]
        ip += 1
        litlen, ip = _ext(block, ip, token >> 4)
        _check(ip + litlen <= len(block), "literals overrun the block")
        out += block[ip:ip + litlen]
        ip += litlen
        st["literal_lengths"].add(litlen)
        st["max_literal"] = max(st["max_literal"], litlen)
        if litlen > 256:
            st["long_literals"] += 1
        if ip == len(block):                             # the last sequence: literals only
            last_seq_has_match = False
            break
        _check(ip + 2 <= len(block), "truncated offset")
        off = block[ip] | block[ip + 1] << 8
        ip += 2
        mlen, ip = _ext(block, ip, token & 15)
        mlen += MINMATCH
        op = len(out) - base
        _check(1 <= off <= len(out), f"offset {off} at output position {op}")
        if off >= mlen:
            out += out[len(out) - off:len(out) - off + mlen]
        else:
            pat = bytes(out[len(out) - off:])
            out += (pat * (mlen // off + 1))[:mlen]
            st["overlapping"] += 1
            if off >= 4:
                st["max_overlap_len_off_ge4"] = max(st["max_overlap_len_off_ge4"], mlen)
            if mlen <= 256 and off <= 3840:
                st["short_overlaps"] += 1
        if off <= 3 and mlen >= 64:
            st["small_offset_runs"].add((off, op & 3))
        st["matches"] += 1
        st["match_lengths"].add(mlen)
        st["min_offset"] = off if st["min_offset"] is None else min(st["min_offset"], off)
        st["max_offset"] = max(st["max_offset"], off)
        if off > 3840:
            st["far_offsets"] += 1
        last_match_start = op
        last_seq_has_match = True
    n = len(out) - base
    _check(not last_seq_has_match, "the last sequence has a match")
    _check(n <= max_len, "block decodes past the block maximum")
    if last_match_start is not None:
        _check(litlen >= LASTLITERALS, f"the last {litlen} bytes are literals, fewer than {LASTLITERALS}")
        _check(last_match_start + MFLIMIT <= n, f"the last match starts {n - last_match_start} bytes before the end, fewer than {MFLIMIT}")
    if expected_len is not None:
        _check(n == expected_len, f"block decodes to {n} bytes, expected {expected_len}")
    return bytes(out[base:]), st


def merge_stats(a: dict, b: dict) -> dict:
    out = dict(a)
    for k, v in b.items():
        if isinstance(v, set):
            out[k] = a[k] | v
        elif k == "min_offset":
            out[k] = v if a[k] is None else (a[k] if v is None else min(a[k], v))
        elif k.startswith("max"):
            out[k] = max(a[k], v)
        else:
            out[k] = a[k] + v
    return out
