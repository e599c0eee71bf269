"""CPU checks of the device's ZSTD page decoder (zstd_dec.cuh), run on the host through auron_b200_zstd_decompress: a corpus of
libzstd frames over levels, strategies, frame flags, literal modes, data shapes and sizes plus hand-built frames, byte for byte
against libzstd's ZSTD_decompress; a header classifier that asserts what the corpus covers; and a seeded mutation fuzz with the
input between inaccessible pages and guard bytes around the output."""
import ctypes as C
import mmap
import random

import numpy as np
import pytest

from auron_b200 import runtime
import zstd_frames as Z

_L = None


def _lib():
    global _L
    if _L is None:
        _L = runtime.lib()
        _L.auron_b200_zstd_decompress.restype = C.c_int64
        _L.auron_b200_zstd_decompress.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        _L.auron_b200_last_error.restype = C.c_char_p
    return _L


class _Fenced:
    """`data` placed right before an inaccessible page (and after one), so that a read past either end faults."""

    def __init__(self, cap):
        page = mmap.PAGESIZE
        self.body = (cap + page - 1) // page * page
        self.m = mmap.mmap(-1, self.body + 2 * page, prot=mmap.PROT_READ | mmap.PROT_WRITE)
        self.base = C.addressof(C.c_char.from_buffer(self.m))
        libc = C.CDLL(None)
        libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
        assert libc.mprotect(self.base, page, 0) == 0
        assert libc.mprotect(self.base + page + self.body, page, 0) == 0
        self.page = page

    def put(self, data):
        start = self.page + self.body - len(data)
        self.m[start:start + len(data)] = data
        return self.base + start


_GUARD = 64


def native(frame, cap, fence=None):
    """Decode with the engine's decoder: (bytes or None, the guard bytes were intact)."""
    f = fence or _Fenced(len(frame) + 1)
    src = f.put(frame)
    out = C.create_string_buffer(b"\xa5" * (cap + 2 * _GUARD))
    r = _lib().auron_b200_zstd_decompress(src, len(frame), C.addressof(out) + _GUARD, cap)
    raw = out.raw
    intact = raw[:_GUARD] == b"\xa5" * _GUARD and raw[_GUARD + cap:_GUARD + cap + _GUARD] == b"\xa5" * _GUARD
    if r < 0:
        assert _lib().auron_b200_last_error()
        return None, intact
    assert 0 <= r <= cap
    return raw[_GUARD:_GUARD + r], intact


def _check(frame, data, cap=None):
    cap = len(data) if cap is None else cap
    ref = Z.decompress(frame, cap)
    assert ref == data
    got, intact = native(frame, cap)
    assert intact
    assert got == ref


def _corpus():
    out = []   # (name, frame, data)
    sh = Z.shapes(300_000, 1)
    for lvl in list(range(-7, 0)) + list(range(1, 23)):
        name = ("text", "int64", "dict_idx", "runs", "noisy", "period")[lvl % 6]
        d = sh[name][:60_000 + 997 * (lvl + 7)]
        out.append(("level%d_%s" % (lvl, name), Z.compress(d, level=lvl), d))
    for strategy in range(1, 10):
        for name in ("text", "int64", "dict_idx"):
            d = sh[name][:150_000]
            out.append(("strategy%d_%s" % (strategy, name), Z.compress(d, level=5, strategy=strategy), d))
    for name, d in sh.items():
        for lm in (1, 2):   # Huffman literals forced on / raw literals
            out.append(("litmode%d_%s" % (lm, name), Z.compress(d, level=3, literal_mode=lm), d))
        out.append(("window10_%s" % name, Z.compress(d, level=9, window_log=10), d))
        out.append(("ldm_%s" % name, Z.compress(d + d, level=12, ldm=1, window_log=20), d + d))
        out.append(("nochecksum_nosize_%s" % name, Z.compress(d, level=3, checksum=0, content_size=0), d))
        out.append(("checksum_%s" % name, Z.compress(d, level=3, checksum=1), d))
        out.append(("smallblocks_%s" % name, Z.compress(d, level=3, target_cblock=1340), d))
    for n in (0, 1, 2, 5, 6, 7, 131_071, 131_072, 131_073, 262_144 + 7):
        d = (sh["text"] * 2)[:n]
        out.append(("size%d" % n, Z.compress(d, level=3, checksum=1), d))
    big = np.random.default_rng(9).integers(0, 1 << 20, 1 << 20).astype(np.int64)
    big.sort()
    d = big.tobytes()[:5_000_000]
    out.append(("multi_mb_level1", Z.compress(d, level=1), d))
    out.append(("multi_mb_level19", Z.compress(d[:2_000_000], level=19), d[:2_000_000]))
    # hand-built: raw and RLE blocks, several frames, skippable frames
    t = sh["text"][:200_000]
    out.append(("raw_blocks", Z.raw_frame(t), t))
    out.append(("raw_blocks_checksum", Z.raw_frame(t[:1000], block_size=300, checksum=True), t[:1000]))
    out.append(("rle_blocks", Z.rle_frame(7, 300_000, pieces=3), bytes([7]) * 300_000))
    out.append(("empty_raw_block", Z.raw_frame(b""), b""))
    a, b = sh["int64"][:40_000], sh["runs"][:24_000]
    out.append(("multi_frame", Z.compress(a, level=3) + Z.raw_frame(b) + Z.compress(b, level=19, checksum=1), a + b + b))
    out.append(("skippable", Z.skippable(b"x" * 17) + Z.compress(a, level=3) + Z.skippable(b"", 15) + Z.compress(b, level=1) + Z.skippable(b"tail", 3),
                a + b))
    out.append(("only_skippable", Z.skippable(b"abc"), b""))
    for name, f in (("rle_literals", Z.rle_literals_frame()), ("many_sequences", Z.many_sequences_frame())):
        d = Z.decompress(f, 1 << 20)
        assert d is not None, name
        out.append((name, f, d))
    return out


_CORPUS = None


def corpus():
    global _CORPUS
    if _CORPUS is None:
        _CORPUS = _corpus()
    return _CORPUS


def test_libzstd_version():
    assert Z.lib().ZSTD_versionNumber() >= 10500


def test_corpus_matches_libzstd():
    for name, frame, data in corpus():
        try:
            _check(frame, data)
        except AssertionError:
            raise AssertionError("corpus frame " + name) from None


def test_corpus_covers_every_case():
    st = {}
    for _, frame, _ in corpus():
        Z.classify(frame, st)
    want = ["frame:zstd", "frame:skippable", "frame:multi_block", "single_segment:0", "single_segment:1", "checksum:0", "checksum:1",
            "fcs:0", "fcs:1", "fcs:2", "fcs:4", "block:raw", "block:rle", "block:compressed",
            "lit:raw", "lit:rle", "lit:compressed", "lit:treeless", "lit_size_format:1", "lit_size_format:2", "lit_size_format:3",
            "lit_size_format:4", "lit_size_format:5", "lit_streams:1", "lit_streams:4", "huf_tree:direct", "huf_tree:fse",
            "seq_count:0", "seq_count:1byte", "seq_count:2byte", "seq_count:3byte"]
    for t in ("ll", "of", "ml"):
        want += ["%s:%s" % (t, m) for m in ("predefined", "rle", "fse", "repeat")]
    missing = [k for k in want if k not in st]
    assert not missing, (missing, sorted(st.items()))


def test_output_must_fit():
    d = Z.shapes(50_000, 3)["text"]
    frame = Z.compress(d, level=3)
    got, intact = native(frame, len(d) - 1)
    assert got is None and intact
    got, intact = native(frame, len(d) + 100)   # room to spare: the bytes written are returned
    assert got == d and intact


@pytest.mark.parametrize("case", ["bad_magic", "reserved_bit", "dict_id", "wrong_checksum", "wrong_content_size", "trailing_bytes",
                                  "reserved_block", "truncated", "window_log"])
def test_rejects_like_libzstd(case):
    d = Z.shapes(20_000, 4)["int64"]
    f = bytearray(Z.compress(d, level=3, checksum=1))
    if case == "bad_magic":
        f[0] ^= 1
    elif case == "reserved_bit":
        f[4] |= 0x08
    elif case == "dict_id":
        f = bytearray(Z.MAGIC + bytes([0x21, 0x10, 5]) + Z.block(0, b"abcde", True))   # single segment, 1-byte dictionary id 16
        d = b"abcde"
    elif case == "wrong_checksum":
        f[-1] ^= 0x40
    elif case == "wrong_content_size":
        f = bytearray(Z.frame_header(len(d) + 1)) + Z.raw_frame(d)[len(Z.frame_header(len(d))):]
    elif case == "trailing_bytes":
        f += b"\x00\x01"
    elif case == "reserved_block":
        f = bytearray(Z.frame_header(None) + bytes([0x07, 0, 0]))
    elif case == "truncated":
        f = f[:-5]
    elif case == "window_log":
        f = bytearray(Z.MAGIC + bytes([0x00, 22 << 3]) + Z.block(0, b"ab", True))
        d = b"ab"
    assert Z.decompress(bytes(f), len(d)) is None
    got, intact = native(bytes(f), len(d))
    assert got is None and intact


def test_dictionary_id_zero_is_accepted():
    f = Z.MAGIC + bytes([0x21, 0x00, 5]) + Z.block(0, b"abcde", True)
    assert Z.decompress(f, 5) == b"abcde"
    assert native(f, 5) == (b"abcde", True)


def test_mutation_fuzz():
    """Seeded mutants of small frames: never a read or write outside the buffers, never a mutant accepted that libzstd rejects, the
    same bytes wherever both accept.  The one disagreement allowed: libzstd's double-symbol Huffman decoder accepts a literal stream
    whose last code runs past the stream's start (it clamps the bit count), which RFC 8878 does not allow; such mutants decode to
    bytes that differ from the original data, so they are corrupt pages, and the engine rejects them."""
    rng = random.Random(20261018)
    bases = []
    for name, d in Z.shapes(6_000, 2).items():
        for lvl in (-3, 1, 3, 9, 19):
            for lm in (0, 2):
                f = Z.compress(d, level=lvl, literal_mode=lm, target_cblock=1500 if lvl == 3 else 0, checksum=1 if lvl == 9 else 0)
                bases.append((f, d))
    bases.append((Z.raw_frame(b"0123456789" * 50, block_size=128, checksum=True), b"0123456789" * 50))
    bases.append((Z.skippable(b"zz") + Z.rle_frame(3, 500, 2), bytes([3]) * 500))
    fence = _Fenced(16_384)
    counts = {"agree_accept": 0, "agree_reject": 0, "lenient_huffman": 0}
    for it in range(30_000):
        frame, data = bases[rng.randrange(len(bases))]
        b = bytearray(frame)
        k = rng.random()
        if k < 0.55:
            for _ in range(rng.randint(1, 3)):
                i = rng.randrange(len(b))
                b[i] ^= 1 << rng.randrange(8)
        elif k < 0.7:
            b = b[:rng.randrange(len(b))]
        elif k < 0.85:
            b[rng.randrange(len(b))] = rng.randrange(256)
        else:   # a size field: block header or literals / sequences header bytes near a block start
            i = rng.randrange(min(len(b), 64))
            b[i] = (b[i] + rng.choice((1, -1, 2, 128))) & 0xFF
        b = bytes(b)
        cap = len(data) + rng.choice((0, 0, 0, 7))
        ref = Z.decompress(b, cap)
        got, intact = native(b, cap, fence)
        assert intact, it
        if ref is None:
            assert got is None, it
            counts["agree_reject"] += 1
        elif got is None:
            assert ref != data, it
            counts["lenient_huffman"] += 1
        else:
            assert got == ref, it
            counts["agree_accept"] += 1
    assert counts["agree_accept"] > 5_000 and counts["agree_reject"] > 5_000, counts
    assert counts["lenient_huffman"] < 0.05 * 30_000, counts
