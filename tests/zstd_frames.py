"""ZSTD test data without a zstd Python module: libzstd 1.5.5 (``libzstd.so.1``) driven through ctypes, hand-built frames for the
block and frame shapes its compressor does not emit, and a classifier that reads only the header bits of a frame (block types,
literals sections, Huffman tree descriptions, sequence counts and table modes) so that tests can assert what a corpus covers."""
import ctypes as C
import struct

import numpy as np

_Z = None

# ZSTD_cParameter values of zstd.h (1.5.5)
LEVEL, WINDOW_LOG, STRATEGY, LDM, CONTENT_SIZE, CHECKSUM = 100, 101, 107, 160, 200, 201
LITERAL_MODE, TARGET_CBLOCK = 1002, 1003   # experimental: ZSTD_c_literalCompressionMode, ZSTD_c_targetCBlockSize


def lib():
    global _Z
    if _Z is None:
        z = C.CDLL("libzstd.so.1")
        z.ZSTD_compressBound.restype = C.c_size_t
        z.ZSTD_compressBound.argtypes = [C.c_size_t]
        z.ZSTD_createCCtx.restype = C.c_void_p
        z.ZSTD_freeCCtx.argtypes = [C.c_void_p]
        z.ZSTD_CCtx_setParameter.restype = C.c_size_t
        z.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
        z.ZSTD_compress2.restype = C.c_size_t
        z.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        z.ZSTD_decompress.restype = C.c_size_t
        z.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        z.ZSTD_isError.restype = C.c_uint
        z.ZSTD_isError.argtypes = [C.c_size_t]
        z.ZSTD_versionNumber.restype = C.c_uint
        _Z = z
    return _Z


def compress(data, **params):
    """ZSTD_compress2 with the given parameters (names: level, window_log, strategy, ldm, content_size, checksum, literal_mode,
    target_cblock); returns None when libzstd refuses a parameter."""
    z = lib()
    cctx = z.ZSTD_createCCtx()
    try:
        ids = {"level": LEVEL, "window_log": WINDOW_LOG, "strategy": STRATEGY, "ldm": LDM, "content_size": CONTENT_SIZE,
               "checksum": CHECKSUM, "literal_mode": LITERAL_MODE, "target_cblock": TARGET_CBLOCK}
        for k, v in params.items():
            if z.ZSTD_isError(z.ZSTD_CCtx_setParameter(cctx, ids[k], int(v))):
                return None
        cap = z.ZSTD_compressBound(len(data))
        dst = C.create_string_buffer(cap)
        r = z.ZSTD_compress2(cctx, dst, cap, data, len(data))
        assert not z.ZSTD_isError(r)
        return dst.raw[:r]
    finally:
        z.ZSTD_freeCCtx(cctx)


def decompress(frame, cap):
    """libzstd's ZSTD_decompress into a buffer of `cap` bytes: the bytes, or None when it rejects the input."""
    z = lib()
    dst = C.create_string_buffer(max(cap, 1))
    r = z.ZSTD_decompress(dst, cap, frame, len(frame))
    return None if z.ZSTD_isError(r) else dst.raw[:r]


# ---------------------------------------------------------------------------------------------------------- hand-built frames
MAGIC = struct.pack("<I", 0xFD2FB528)


def frame_header(content_size=None, checksum=False, window_log=17):
    if content_size is None:
        return MAGIC + bytes([(1 << 2 if checksum else 0), (window_log - 10) << 3])
    if content_size < 256:
        return MAGIC + bytes([0x20 | (1 << 2 if checksum else 0), content_size])   # single segment, 1-byte size
    return MAGIC + bytes([0x80 | 0x20 | (1 << 2 if checksum else 0)]) + struct.pack("<I", content_size)


def block(kind, body, last, size=None):
    """kind 0 raw, 1 RLE (body = one byte, size = its run), 2 compressed"""
    n = size if kind == 1 else len(body)
    h = (n << 3) | (kind << 1) | (1 if last else 0)
    return struct.pack("<I", h)[:3] + body


def raw_frame(data, block_size=1 << 17, checksum=False):
    blocks = [data[i:i + block_size] for i in range(0, len(data), block_size)] or [b""]
    out = frame_header(len(data), checksum)
    for i, b in enumerate(blocks):
        out += block(0, b, i == len(blocks) - 1)
    return out + (struct.pack("<I", xxh64(data) & 0xFFFFFFFF) if checksum else b"")


def rle_frame(byte, n, pieces=1):
    out = frame_header(None)
    each = [n // pieces] * pieces
    each[-1] += n - sum(each)
    for i, k in enumerate(each):
        out += block(1, bytes([byte]), i == pieces - 1, k)
    return out


def rle_literals_frame(byte=ord("q"), sizes=(9, 700)):
    """A frame of compressed blocks whose literals section is RLE (1- and 2-byte size formats) and which carry no sequences."""
    out = frame_header(None)
    for i, n in enumerate(sizes):
        lit = bytes([(n << 3) | 1]) if n < 32 else struct.pack("<H", (n << 4) | (1 << 2) | 1)
        out += block(2, lit + bytes([byte, 0]), i == len(sizes) - 1)
    return out


def many_sequences_frame(nseq=32_600):
    """A raw block "abcd", then one compressed block of `nseq` sequences (the 3-byte sequence count) with RLE tables for LL, OF and
    ML: literal length 0, match length 3, offset code 0 -- repeat offsets 2 and 1 alternately (literal length 0 shifts them), no
    extra bits, so the bit stream is its end mark only.  The raw literals "wxyz" end the block."""
    assert nseq >= 0x7F00
    body = bytes([4 << 3]) + b"wxyz" + bytes([255]) + struct.pack("<H", nseq - 0x7F00) + bytes([0x54, 0, 0, 0, 1])
    return frame_header(None) + block(0, b"abcd", False) + block(2, body, True)


def skippable(payload, nibble=0):
    return struct.pack("<II", 0x184D2A50 | nibble, len(payload)) + payload


def xxh64(data, seed=0):
    P1, P2, P3, P4, P5 = 0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5
    M = (1 << 64) - 1

    def rotl(x, r):
        return ((x << r) | (x >> (64 - r))) & M

    def rnd(acc, v):
        return (rotl((acc + v * P2) & M, 31) * P1) & M

    n, i = len(data), 0
    if n >= 32:
        v = [(seed + P1 + P2) & M, (seed + P2) & M, seed, (seed - P1) & M]
        while i + 32 <= n:
            for k in range(4):
                v[k] = rnd(v[k], struct.unpack_from("<Q", data, i + 8 * k)[0])
            i += 32
        h = (rotl(v[0], 1) + rotl(v[1], 7) + rotl(v[2], 12) + rotl(v[3], 18)) & M
        for k in range(4):
            h = ((h ^ rnd(0, v[k])) * P1 + P4) & M
    else:
        h = (seed + P5) & M
    h = (h + n) & M
    while i + 8 <= n:
        h = (rotl(h ^ rnd(0, struct.unpack_from("<Q", data, i)[0]), 27) * P1 + P4) & M
        i += 8
    if i + 4 <= n:
        h = (rotl(h ^ (struct.unpack_from("<I", data, i)[0] * P1 & M), 23) * P2 + P3) & M
        i += 4
    while i < n:
        h = (rotl(h ^ (data[i] * P5 & M), 11) * P1) & M
        i += 1
    h ^= h >> 33
    h = (h * P2) & M
    h ^= h >> 29
    h = (h * P3) & M
    h ^= h >> 32
    return h


# ---------------------------------------------------------------------------------------------------------- header classifier
def classify(body, stats=None):
    """Walk the frames of `body` by their headers only and count the features seen.  Returns a dict feature -> count."""
    st = stats if stats is not None else {}

    def see(k):
        st[k] = st.get(k, 0) + 1

    i, n = 0, len(body)
    while i + 4 <= n:
        magic = struct.unpack_from("<I", body, i)[0]
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            see("frame:skippable")
            i += 8 + struct.unpack_from("<I", body, i + 4)[0]
            continue
        assert magic == 0xFD2FB528
        see("frame:zstd")
        fhd = body[i + 4]
        fcs_flag, single, checksum, did = fhd >> 6, (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
        see("fcs:%d" % ([single, 2, 4, 8][fcs_flag]))
        see("single_segment:%d" % single)
        see("checksum:%d" % checksum)
        i += 5 + (0 if single else 1) + [0, 1, 2, 4][did] + [single, 2, 4, 8][fcs_flag]
        nblocks = 0
        while True:
            h = body[i] | body[i + 1] << 8 | body[i + 2] << 16
            last, kind, size = h & 1, (h >> 1) & 3, h >> 3
            i += 3
            nblocks += 1
            see("block:" + ["raw", "rle", "compressed"][kind])
            if kind == 2:
                _classify_block(body[i:i + size], see)
            i += 1 if kind == 1 else size
            if last:
                break
        if nblocks > 1:
            see("frame:multi_block")
        i += 4 if checksum else 0
    return st


def _classify_block(b, see):
    lt, sf = b[0] & 3, (b[0] >> 2) & 3
    see("lit:" + ["raw", "rle", "compressed", "treeless"][lt])
    if lt < 2:
        lh = {1: 2, 3: 3}.get(sf, 1)
        see("lit_size_format:%d" % lh)
        size = b[0] >> 3 if lh == 1 else (int.from_bytes(b[:lh], "little") >> 4)
        p = lh + (size if lt == 0 else 1)
    else:
        lh = 3 if sf < 2 else sf + 2
        see("lit_size_format:%d" % lh)
        see("lit_streams:%d" % (1 if sf == 0 else 4))
        h = int.from_bytes(b[:lh], "little")
        bits = {3: 10, 4: 14, 5: 18}[lh]
        csize = (h >> (4 + bits)) & ((1 << bits) - 1)
        if lt == 2:
            see("huf_tree:" + ("direct" if b[lh] >= 128 else "fse"))
        p = lh + csize
    nseq = b[p]
    if nseq == 0:
        see("seq_count:0")
        return
    if nseq < 128:
        see("seq_count:1byte")
        p += 1
    elif nseq < 255:
        see("seq_count:2byte")
        p += 2
    else:
        see("seq_count:3byte")
        p += 3
    modes = b[p]
    for name, sh in (("ll", 6), ("of", 4), ("ml", 2)):
        see("%s:%s" % (name, ["predefined", "rle", "fse", "repeat"][(modes >> sh) & 3]))


# ---------------------------------------------------------------------------------------------------------- data shapes
def shapes(n, seed):
    rng = np.random.default_rng(seed)
    words = [b"select", b"from", b"where", b"store_sales", b"ss_item_sk", b"group", b"by", b"order", b"date_dim", b"1998", b"customer"]
    text = b" ".join(words[k] for k in rng.integers(0, len(words), n // 4 + 1))[:n]
    runs = np.repeat(rng.integers(0, 4, n // 64 + 1).astype(np.uint8), rng.integers(1, 200, n // 64 + 1))[:n].tobytes()
    runs = (runs + bytes(n))[:n]
    period = (bytes(rng.integers(0, 256, 7).astype(np.uint8)) * (n // 7 + 1))[:n]
    noisy = rng.integers(0, 256, n).astype(np.uint8)
    noisy[rng.random(n) < 0.1] = 0
    ints = np.cumsum(rng.integers(0, 1000, n // 8 + 1)).astype(np.int64).tobytes()[:n]
    dict_idx = np.packbits(np.unpackbits(rng.integers(0, 1 << 11, n // 2 + 1).astype(">u2").view(np.uint8))[:n * 8]).tobytes()[:n]
    return {"text": text, "runs": runs, "period": period, "noisy": noisy.tobytes(), "int64": ints, "dict_idx": dict_idx}
