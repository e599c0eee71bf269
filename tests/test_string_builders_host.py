"""CPU checks of md5 / sha2 and the string constructors (concat, concat_ws, repeat, space): the digest code the device runs,
executed on the host through auron_b200_digest_hex, against hashlib; and the planner, through runtime.explain, accepting every
supported shape and naming the function in every rejected one.

Semantics restated from the reference (paths relative to native-engine/datafusion-ext-functions/src):
  * Spark_MD5 / Spark_Sha224/256/384/512: digest of a utf8 or binary value's bytes, lowercase hex, NULL -> NULL
    (spark_crypto.rs:33-105); goldens spark_crypto.rs:140-208
  * Spark_StringConcat: NULL if any argument is NULL (spark_strings.rs:117-192)
  * Spark_StringConcatWs: literal utf8 separator, NULL arguments skipped (:194-319)
  * Spark_StringRepeat: literal int32 count; NULL count -> NULL, n < 0 -> "" (:75-91)
  * Spark_StringSpace: int32 n; NULL -> NULL, n < 0 -> "" (:65-73)
"""
import ctypes as C
import hashlib
import os

import pyarrow as pa
import pytest

from auron_b200 import proto as P
from auron_b200 import runtime

ALGS = {128: hashlib.md5, 224: hashlib.sha224, 256: hashlib.sha256, 384: hashlib.sha384, 512: hashlib.sha512}


def _digest(alg: int, data: bytes) -> str:
    L = runtime.lib()
    L.auron_b200_digest_hex.restype = C.c_int
    L.auron_b200_digest_hex.argtypes = [C.c_int32, C.c_char_p, C.c_int64, C.c_char_p]
    out = C.create_string_buffer(128)
    n = L.auron_b200_digest_hex(alg, data, len(data), out)
    assert n > 0, runtime._err()
    return out.raw[:n].decode()


def test_digest_matches_hashlib_at_every_padding_boundary():
    # lengths 0..300 cross the one-/two-block boundaries of MD5 / SHA-256 (55/56, 63/64, 119/120, 127/128) and SHA-512 (111/112,
    # 127/128, 239/240, 255/256)
    data = bytes((i * 131 + 7) & 0xff for i in range(300))
    for alg, h in ALGS.items():
        for n in range(301):
            assert _digest(alg, data[:n]) == h(data[:n]).hexdigest(), (alg, n)


def test_digest_of_one_megabyte():
    data = os.urandom(1 << 20)
    for alg, h in ALGS.items():
        assert _digest(alg, data) == h(data).hexdigest(), alg


def test_digest_reference_goldens():
    # spark_crypto.rs:140-208: "ABC" as utf8 and bytes 1..6 as binary
    abc, six = b"ABC", bytes([1, 2, 3, 4, 5, 6])
    assert _digest(224, abc) == "107c5072b799c4771f328304cfe1ebb375eb6ea7f35a3aa753836fad"
    assert _digest(256, abc) == "b5d4045c3f466fa91fe2cc6abe79232a1a57cdf104f7a26e716e0a1e2789df78"
    assert _digest(384, abc) == "1e02dc92a41db610c9bcdc9b5935d1fb9be5639116f6c67e97bc1a3ac649753baba7ba021c813e1fe20c0480213ad371"
    assert _digest(512, abc) == ("397118fdac8d83ad98813c50759c85b8c47565d8268bf10da483153b747a74743a58a90e85aa9f705ce6984ffc128db5"
                                 "67489817e4092d050d8a1cc596ddc119")
    assert _digest(224, six) == "4225cbc32d17010d1a440de9e34504c1fae29b8ee5e527e191ff9a82"
    assert _digest(256, six) == "7192385c3c0605de55bb9476ce1d90748190ecb32a8eed7f5207b30cf6a1fe89"
    assert _digest(384, six) == "557cfe660c753b830efa61528fc350ef384a7a4b9d3467c6230049bc59548eb8a404874baff89cb0f9bd18400829fdc2"
    assert _digest(512, six) == ("178d767c364244ede054ebb3cc4af0ac2b307a86fba6a32706ce4f692642674d2ab8f51ee738ecb09bc296918aa85db4"
                                 "8abe28fcaef7aa2da81a618cc6d891c3")
    assert _digest(128, abc) == "902fbdd2b1df0c4f70b4a5d23525e932"
    assert _digest(128, six) == "6ac1e56bc78f031059be7be854522c4c"


def test_digest_rejects_bad_arguments_with_their_own_message():
    L = runtime.lib()
    L.auron_b200_digest_hex.argtypes = [C.c_int32, C.c_char_p, C.c_int64, C.c_char_p]
    out = C.create_string_buffer(128)
    assert L.auron_b200_digest_hex(0, b"x", 1, out) == -1
    assert "unknown digest algorithm 0" in runtime._err()
    assert L.auron_b200_digest_hex(256, b"x", -1, out) == -1
    assert "negative length" in runtime._err()
    assert L.auron_b200_digest_hex(256, None, 3, out) == -1
    assert "null buffer" in runtime._err()
    assert _digest(256, b"") == hashlib.sha256(b"").hexdigest()


# ------------------------------------------------------------------------------------------------------------ planning
SCHEMA = pa.schema([("s", pa.string()), ("b", pa.binary()), ("i", pa.int64()), ("n", pa.int32()), ("d", pa.date32()),
                    ("dec", pa.decimal128(17, 2)), ("f", pa.float64()), ("flag", pa.bool_())])
U = pa.string()


def _fn(name, *args):
    return P.scalar_fn(name, list(args), U)


def _lit(v, t=U):
    return P.lit(v, t)


def _ws(*args):
    return _fn("Spark_StringConcatWs", _lit("|"), *args)


def _project(exprs, src=None):
    src = src or P.ffi_reader(SCHEMA, "t")
    return P.projection(src, exprs, [f"c{i}" for i in range(len(exprs))], [U] * len(exprs))


def _explain(plan):
    return runtime.explain(P.task_definition(plan))


SUPPORTED = {
    "md5_column": _fn("Spark_MD5", P.col("s")),
    "sha_binary_column": _fn("Spark_Sha256", P.col("b")),
    "sha224_of_upper": _fn("Spark_Sha224", _fn("Upper", P.col("s"))),
    "sha384_of_substr": _fn("Spark_Sha384", P.scalar_fn("Substr", [P.col("s"), _lit(2, pa.int64()), _lit(3, pa.int64())], U)),
    "sha512_of_cast": _fn("Spark_Sha512", P.cast(P.col("i"), U)),
    "concat": _fn("Spark_StringConcat", _lit("store"), P.col("s"), P.cast(P.col("i"), U)),
    "concat_null_literal": _fn("Spark_StringConcat", P.col("s"), _lit(None)),
    "concat_ws": _ws(P.cast(P.col("i"), U), P.col("s"), P.cast(P.col("d"), U), P.cast(P.col("dec"), U), _fn("Upper", P.col("s")),
                     P.cast(P.col("flag"), U), _lit(None)),
    "concat_ws_null_separator": _fn("Spark_StringConcatWs", _lit(None), P.col("s")),
    "concat_ws_of_case_and_coalesce": _ws(P.case([(P.is_null(P.col("s")), _lit("none"))], P.col("s")),
                                          P.scalar_fn("Coalesce", [P.col("s"), _lit("-")], U)),
    "repeat": _fn("Spark_StringRepeat", P.col("s"), _lit(3, pa.int32())),
    "repeat_null_count": _fn("Spark_StringRepeat", P.col("s"), _lit(None, pa.int32())),
    "repeat_cast": _fn("Spark_StringRepeat", P.cast(P.col("n"), U), _lit(2, pa.int32())),
    "space": _fn("Spark_StringSpace", P.col("n")),
    "md5_of_concat_ws": _fn("Spark_MD5", _ws(P.cast(P.col("i"), U), P.col("s"))),
    "sha2_of_concat": _fn("Spark_Sha256", _fn("Spark_StringConcat", P.col("s"), P.col("s"))),
    "declared_type_wrapper": P.try_cast(_fn("Spark_MD5", P.col("s")), U),
}


@pytest.mark.parametrize("shape", sorted(SUPPORTED))
def test_supported_shapes_plan(shape):
    plan = _explain(_project([SUPPORTED[shape], P.col("i")]))["plan"]
    assert plan["op"] == "ProjectExec"
    assert plan["schema"][0][1] in ("Utf8", "utf8"), plan["schema"]


def test_all_shapes_in_one_projection_and_as_keys():
    # every constructor / digest in one program: the hidden digest arguments count against the program's output slots
    _explain(_project(list(SUPPORTED.values())))
    src = P.ffi_reader(SCHEMA, "t")
    key = _fn("Spark_MD5", _ws(P.col("s"), P.cast(P.col("i"), U)))
    _explain(P.agg(src, [key], ["k"], [P.agg_expr("COUNT", [P.col("i")], pa.int64())], ["c"], ["PARTIAL"]))
    _explain(P.shuffle_writer(src, P.hash_repartition([_fn("Spark_StringConcat", P.col("s"), P.col("s"))], 4), "/tmp/x.data", "/tmp/x.index"))


REJECTED = {
    "non_literal_separator": ("Spark_StringConcatWs", _fn("Spark_StringConcatWs", P.col("s"), P.col("s"))),
    "list_argument": ("Spark_StringConcatWs", _ws(P.lit(["a", "b"], pa.list_(pa.string())))),
    "non_literal_repeat_count": ("Spark_StringRepeat", _fn("Spark_StringRepeat", P.col("s"), P.col("n"))),
    "digest_in_substr": ("Spark_MD5", P.scalar_fn("Substr", [_fn("Spark_MD5", P.col("s")), _lit(1, pa.int64()), _lit(4, pa.int64())], U)),
    "digest_in_upper": ("Spark_Sha256", _fn("Upper", _fn("Spark_Sha256", P.col("s")))),
    "digest_in_comparison": ("Spark_MD5", P.binary("Eq", _fn("Spark_MD5", P.col("s")), _lit("x"))),
    "digest_of_digest": ("Spark_MD5", _fn("Spark_Sha256", _fn("Spark_MD5", P.col("s")))),
    "constructor_in_constructor": ("Spark_StringSpace", _fn("Spark_StringConcat", P.col("s"), _fn("Spark_StringSpace", P.col("n")))),
    "constructor_in_case": ("Spark_StringConcat", P.case([(P.is_null(P.col("s")), _fn("Spark_StringConcat", P.col("s")))], P.col("s"))),
    "md5_of_int": ("Spark_MD5", _fn("Spark_MD5", P.col("i"))),
    "float_piece": ("Spark_StringConcat", _fn("Spark_StringConcat", P.col("s"), P.cast(P.col("f"), U))),
    "space_of_int64": ("Spark_StringSpace", _fn("Spark_StringSpace", P.col("i"))),
    "space_of_cast_int64": ("Spark_StringSpace", _fn("Spark_StringSpace", P.cast(P.col("i"), U))),
    "space_of_cast_int32": ("Spark_StringSpace", _fn("Spark_StringSpace", P.cast(P.col("n"), U))),
    "space_of_string": ("Spark_StringSpace", _fn("Spark_StringSpace", P.col("s"))),
}


@pytest.mark.parametrize("shape", sorted(REJECTED))
def test_rejected_shapes_name_the_function(shape):
    name, expr = REJECTED[shape]
    with pytest.raises(runtime.AuronError, match=name):
        _explain(_project([expr]))


def test_constructor_in_a_filter_is_rejected():
    src = P.ffi_reader(SCHEMA, "t")
    pred = P.binary("Eq", _fn("Spark_StringConcat", P.col("s"), _lit("x")), _lit("ax"))
    with pytest.raises(runtime.AuronError, match="Spark_StringConcat"):
        _explain(P.filter_(src, [pred]))
