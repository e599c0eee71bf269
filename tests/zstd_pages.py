"""Hand-built Parquet files whose page bodies are given compressed bytes: one required INT64 PLAIN column of v2 data pages under
the ZSTD or LZ4_RAW codec.  Any ZSTD body whose output is a multiple of 8 bytes is a valid page, so every frame of the CPU
corpus (tests/test_zstd_host.py) can be scanned on the device and compared with np.frombuffer(output, int64)."""
import struct

from parquet_pages import _BIN, _I32, _I64, _LIST, _STRUCT, _struct

CODEC_ZSTD, CODEC_LZ4_RAW = 6, 7


def write(path, bodies, codec=CODEC_ZSTD, name="c"):
    """bodies: [(compressed bytes, uncompressed length)], one data page each (the length a multiple of 8)."""
    body = bytearray()
    rows = 0
    for comp, n in bodies:
        assert n % 8 == 0
        k = n // 8
        hdr = _struct([(1, _I32, 3), (2, _I32, n), (3, _I32, len(comp)),
                       (8, _STRUCT, [(1, _I32, k), (2, _I32, 0), (3, _I32, k), (4, _I32, 0), (5, _I32, 0), (6, _I32, 0)])])
        body += hdr + comp
        rows += k
    meta = [(1, _I32, 2), (2, _LIST, (_I32, [0, 3])), (3, _LIST, (_BIN, [name.encode()])), (4, _I32, codec), (5, _I64, rows),
            (6, _I64, len(body)), (7, _I64, len(body)), (9, _I64, 4)]
    footer = _struct([
        (1, _I32, 2),
        (2, _LIST, (_STRUCT, [[(4, _BIN, b"schema"), (5, _I32, 1)], [(1, _I32, 2), (3, _I32, 0), (4, _BIN, name.encode())]])),
        (3, _I64, rows),
        (4, _LIST, (_STRUCT, [[(1, _LIST, (_STRUCT, [[(2, _I64, 4), (3, _STRUCT, meta)]])), (2, _I64, len(body)), (3, _I64, rows)]])),
    ])
    with open(path, "wb") as f:
        f.write(b"PAR1" + bytes(body) + footer + struct.pack("<I", len(footer)) + b"PAR1")
    return rows
