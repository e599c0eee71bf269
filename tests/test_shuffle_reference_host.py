"""Pins the plain-Python shuffle references of shuffle_reference.py (CPU only): the batch layout against the oracle's port of
write_batch / read_batch, xxh32 against published vectors, and the LZ4 frame walker and strict block decoder against Arrow's
LZ4 frame reader and liblz4 (pyarrow's lz4_raw codec) -- so the GPU tests that use them measure the engine, not the reference."""
import random
import struct

import pyarrow as pa
import pytest

import key_reference as R
import oracle
import shuffle_reference as S
from test_gpu_key_edges import ARROW, BITMAPS, from_arrow, to_arrow


def _sliced(t, n, seed, bitmap, off=3):
    full = R.edge_column(t, n + off + 8, seed, null_rate=0.05 if bitmap == "nulls" else 0.0)
    return full[off:off + n], to_arrow(full, t, bitmap != "no_bitmap").slice(off, n)


@pytest.mark.parametrize("t", R.TYPES)
def test_write_batch_matches_the_oracle(t):
    # the oracle's rule: has_nulls = 1 exactly when the array holds a NULL; arrays sliced at offset 3 (validity re-based to bit 0)
    for n in (0, 1, 7, 8, 9, 129):
        for i, bitmap in enumerate(BITMAPS):
            vals, arr = _sliced(t, n, seed=10 * n + i, bitmap=bitmap)
            assert arr.offset == 3
            exp = oracle.serde_write_batch(pa.record_batch([arr], names=["c"]))
            assert S.write_batch([(t, vals)], [arr.null_count > 0]) == exp, (t, n, bitmap)


def test_write_batch_of_every_type_and_null_columns_matches_the_oracle():
    # a Null column writes nothing (batch_serde.rs write_array: DataType::Null => {}), so the oracle's batch without it is the same bytes
    for n in (0, 1, 9, 129):
        cols, arrs = [], []
        for i, t in enumerate(R.TYPES):
            vals, arr = _sliced(t, n, seed=n + i, bitmap=BITMAPS[i % 3])
            cols.append((t, vals))
            arrs.append(arr)
        got = S.write_batch(cols[:5] + [("null", [None] * n)] + cols[5:] + [("null", [None] * n)],
                            [a.null_count > 0 for a in arrs[:5]] + [None] + [a.null_count > 0 for a in arrs[5:]] + [None])
        assert got == oracle.serde_write_batch(pa.record_batch(arrs, names=list(R.TYPES)))
    assert S.write_batch([("null", [None] * 300)], [None]) == S.write_len(300) == oracle.write_len(300)


def test_varint_row_counts():
    for v in (0, 1, 127, 128, 129, 16383, 16384, 16385, 2**21 - 1, 2**21, 2**35 + 7):
        assert S.write_len(v) == oracle.write_len(v)
        assert S.read_len(S.write_len(v) + b"\x55", 0) == (v, len(S.write_len(v)))
    assert [len(S.write_len(v)) for v in (127, 128, 16383, 16384)] == [1, 2, 2, 3]


def test_read_sections_inverts_write_batch():
    schema = list(R.TYPES[:7]) + ["null"] + list(R.TYPES[7:])
    payload, exp = b"", []
    for b, n in enumerate((1, 0, 9, 129, 8)):
        cols = [(t, [None] * n if t == "null" else R.edge_column(t, n + 1, seed=b * 31 + i)[:n]) for i, t in enumerate(schema)]
        hn = [None if t == "null" else (i + b) % 2 == 0 or any(v is None for v in vals) for i, (t, vals) in enumerate(cols)]
        start = len(payload)
        payload += S.write_batch(cols, hn)
        exp.append((start, len(payload), n, [v for _, v in cols], [None if h is None else int(h) for h in hn]))
    got = S.read_sections(payload, schema)
    assert [(g["start"], g["end"], g["n"], g["cols"], g["has_nulls"]) for g in got] == exp
    # the oracle's reader takes the same bytes (the Null column has no oracle reader: read without it)
    for g in got:
        if g["n"] == 0:
            continue
        fields = [(t, c) for t, c in zip(schema, g["cols"]) if t != "null"]
        sub = S.write_batch(fields, [h for t, h in zip(schema, g["has_nulls"]) if t != "null"])
        rb, end = oracle.serde_read_batch(sub, pa.schema([(f"c{i}", ARROW[t]) for i, (t, _) in enumerate(fields)]))
        assert end == len(sub)
        assert [from_arrow(rb.column(i), t) for i, (t, _) in enumerate(fields)] == [c for _, c in fields]


def test_read_sections_rejects_nonzero_padding_and_truncation():
    good = S.write_batch([("bool", [True, None, False])], [1])
    assert good == bytes([3, 1, 0b101, 0b001])
    with pytest.raises(AssertionError):
        S.read_sections(bytes([3, 1, 0b1101, 0b001]), ["bool"])          # validity padding bit 3 set
    with pytest.raises(AssertionError):
        S.read_sections(bytes([3, 1, 0b101, 0b1001]), ["bool"])          # value padding bit 3 set
    with pytest.raises(AssertionError):
        S.read_sections(S.write_batch([("int64", [1, 2])], [0])[:-1], ["int64"])


def test_xxh32_known_vectors():
    assert S.xxh32(b"") == 0x02CC5D05
    assert S.xxh32(b"a") == 0x550D7456
    assert S.xxh32(b"abc") == 0x32D153FF
    assert S.xxh32(b"Nobody inspects the spammish repetition") == 0xE2293B2F
    assert S.header_checksum(bytes([0x60, 0x40])) == 0x82         # the header this engine's GPU frames carry (shuffle_writer.cc)


def _arrow_lz4f(data: bytes) -> bytes:
    sink = pa.BufferOutputStream()
    with pa.CompressedOutputStream(sink, "lz4") as z:
        z.write(data)
    return sink.getvalue().to_pybytes()


def _arrow_lz4f_read(frame: bytes) -> bytes:
    return pa.CompressedInputStream(pa.BufferReader(frame), "lz4").read()


def _payloads():
    rng = random.Random(5)
    rand = bytes(rng.randrange(256) for _ in range(200_000))
    cols = [(t, R.edge_column(t, 3000, seed=i)) for i, t in enumerate(R.TYPES)]
    batch = S.write_batch(cols, [1] * len(cols))
    return {"zeros": bytes(150_000), "random": rand, "period3": b"xyz" * 70_000, "batch": batch * 3,
            "mixed": b"".join(rand[i:i + 300] + bytes([i % 7]) * (i % 500) for i in range(0, 60_000, 300)), "short": b"0123456789abc"}


@pytest.mark.parametrize("name", ["zeros", "random", "period3", "batch", "mixed", "short"])
def test_frame_walker_and_block_decoder_match_arrow_on_linked_frames(name):
    data = _payloads()[name]
    frame = _arrow_lz4f(data)
    info = S.lz4_frame_blocks(struct.pack("<I", len(frame)) + frame)
    assert info["linked"] and info["block_max"] == 64 << 10
    assert S.lz4_frame_decode(info) == _arrow_lz4f_read(frame) == data


def _lz4_raw(raw: bytes) -> bytes:
    return pa.compress(raw, codec="lz4_raw", asbytes=True)


@pytest.mark.parametrize("name", ["zeros", "random", "period3", "batch", "mixed", "short"])
def test_independent_frames_from_lz4_raw_blocks(name):
    # frames shaped like lz4_flex's FrameEncoder: independent 64 KB blocks, a short last block, stored blocks where liblz4 did not shrink
    data = _payloads()[name]
    chunks = [data[o:o + 65536] for o in range(0, len(data), 65536)]
    frame = S.lz4_frame([(c, _lz4_raw(c)) for c in chunks])
    assert _arrow_lz4f_read(frame) == data                      # Arrow's LZ4F reader accepts the hand-assembled frame
    info = S.lz4_frame_blocks(struct.pack("<I", len(frame)) + frame)
    assert not info["linked"] and len(info["blocks"]) == len(chunks)
    for (stored, blk), raw in zip(info["blocks"], chunks):
        assert stored == (len(_lz4_raw(raw)) >= len(raw))
        if not stored:
            got, _ = S.lz4_block_decode(blk, expected_len=len(raw))
            assert got == raw == bytes(pa.decompress(blk, decompressed_size=len(raw), codec="lz4_raw"))
    assert S.lz4_frame_decode(info) == data
    if name == "random":
        assert all(s for s, _ in info["blocks"])


def _seq(lits: bytes, off=None, mlen=None) -> bytes:
    """one hand-made sequence: token, literal length extension, literals, [offset, match length extension]"""
    def ext(v):
        if v < 15:
            return b""
        v -= 15
        return b"\xff" * (v // 255) + bytes([v % 255])
    ml = None if mlen is None else mlen - 4
    token = (min(len(lits), 15) << 4) | (0 if ml is None else min(ml, 15))
    out = bytes([token]) + ext(len(lits)) + lits
    if off is not None:
        out += struct.pack("<H", off) + ext(ml)
    return out


def test_strict_decoder_accepts_well_formed_hand_made_blocks():
    lit270 = bytes(range(256)) + b"0123456789abcd"
    for blk, exp in [(_seq(b"abcdefgh", 8, 8) + _seq(b"12345"), b"abcdefgh" * 2 + b"12345"),
                     (_seq(b"a", 1, 4 + 15 + 255) + _seq(b"xxxxx"), b"a" * 275 + b"xxxxx"),
                     (_seq(lit270, 270, 8) + _seq(b"12345"), lit270 + lit270[:8] + b"12345"),
                     (_seq(b"q" * 12), b"q" * 12), (_seq(b""), b"")]:
        got, st = S.lz4_block_decode(blk, expected_len=len(exp))
        assert got == exp
        if exp:
            assert bytes(pa.decompress(blk, decompressed_size=len(exp), codec="lz4_raw")) == exp
    assert 270 in S.lz4_block_decode(_seq(lit270, 270, 8) + _seq(b"12345"))[1]["literal_lengths"]
    assert _seq(lit270)[:3] == b"\xf0\xff\x00"                    # 15 + 255: one 255 byte and a final 0


@pytest.mark.parametrize("case", ["ends_with_match", "last_literals_4", "match_starts_11_before_end", "offset_0", "offset_past_start",
                                  "wrong_length", "truncated_literals", "truncated_offset"])
def test_strict_decoder_rejects_broken_blocks(case):
    blk, exp = {
        "ends_with_match": (_seq(b"abcdefgh", 8, 8), 16),
        "last_literals_4": (_seq(b"abcdefgh", 8, 8) + _seq(b"1234"), 20),
        "match_starts_11_before_end": (_seq(b"abcdefghijklmnop", 4, 6) + _seq(b"12345"), 27),   # match at 16 of 27
        "offset_0": (_seq(b"abcdefgh", 0, 8) + _seq(b"12345"), 21),
        "offset_past_start": (_seq(b"abcdefgh", 9, 8) + _seq(b"12345"), 21),
        "wrong_length": (_seq(b"abcdefgh", 8, 8) + _seq(b"12345"), 22),
        "truncated_literals": (_seq(b"abcdefgh")[:-1], 8),
        "truncated_offset": (_seq(b"abcdefgh", 8, 8)[:-1], 16),
    }[case]
    with pytest.raises(AssertionError):
        S.lz4_block_decode(blk, expected_len=exp)
    # the same block, made well-formed, passes: the rule that fired is the one the case breaks
    if case == "match_starts_11_before_end":
        S.lz4_block_decode(_seq(b"abcdefghijklmnop", 4, 6) + _seq(b"123456"), expected_len=28)


def test_frame_walker_rejects_a_bad_header_checksum_and_trailing_bytes():
    frame = S.lz4_frame([(b"abc", _lz4_raw(b"abc"))])
    ok = struct.pack("<I", len(frame)) + frame
    assert S.lz4_frame_blocks(ok)["hc"] == 0x82
    bad = bytearray(ok)
    bad[4 + 6] ^= 1
    with pytest.raises(AssertionError):
        S.lz4_frame_blocks(bytes(bad))
    with pytest.raises(AssertionError):
        S.lz4_frame_blocks(struct.pack("<I", len(frame) + 1) + frame + b"\0")
    assert S.split_streams(ok + ok) == [ok, ok]
    with pytest.raises(AssertionError):
        S.split_streams(ok + ok[:-1])
