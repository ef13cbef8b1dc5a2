"""nestedArrayFormat=ragged (include/tfrgpu.h, RAGGED) without a GPU: the option, the schema lowering and its refusals, and the
restatement in tests/ragged_rows.py, whose bytes upb's tensorflow.Example parses back into the two plain features."""
import ctypes as C
import os
import subprocess

import pytest

import ragged_rows as RR
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native, io
from spark_tfrecord_b200.sqltypes import *  # noqa

X = StructType([StructField("id", LongType(), False), StructField("x", ArrayType(ArrayType(LongType())), True),
                StructField("s", ArrayType(ArrayType(StringType())), False)])


def _create(schema, rt=0, flags=A.TFR_S_RAGGED):
    fields, keep = A.make_fields(schema)
    h = C.c_void_p()
    rc = _native.lib().tfr_schema_create_ex(fields, len(schema), rt, flags, C.byref(h))
    n = _native.lib().tfr_schema_num_fields(h) if rc == 0 else None
    if rc == 0:
        _native.lib().tfr_schema_destroy(h)
    return rc, n, _native.lib().tfr_last_error().decode()


def test_option_values():
    assert io._nested_array_format({}) is False
    assert io._nested_array_format({"nestedArrayFormat": "featureList"}) is False
    assert io._nested_array_format({"nestedArrayFormat": "ragged"}) is True
    with pytest.raises(_native.IllegalArgumentException):
        io._nested_array_format({"nestedArrayFormat": "Ragged"})
    with pytest.raises(_native.IllegalArgumentException):
        io._nested_array_format({"nestedArrayFormat": "ragged", "recordType": "SequenceExample"})
    with pytest.raises(_native.IllegalArgumentException):
        io.DefaultSource().prepareWrite({"nestedArrayFormat": "rowSplits"}, X)
    with pytest.raises(_native.IllegalArgumentException):
        io.DefaultSource().buildReader(X, X, {"nestedArrayFormat": "x"})


def test_schema_flags_and_counts():
    assert _create(X)[:2] == (0, 3)                                 # a ragged field stays one column
    assert _create(X, flags=0)[:2] == (0, 3)
    rc, _, msg = _create(X, rt=1)
    assert rc == A.TFR_E_INVALID_ARG and "SequenceExample" in msg
    assert _create(X, flags=2)[0] == A.TFR_E_INVALID_ARG
    assert _create(X, rt=2)[0] == 0                                 # ByteArray ignores it
    sv = StructType([StructField("v", VectorUDT()), StructField("x", ArrayType(ArrayType(IntegerType())))])
    fields, keep = A.make_fields(sv, "sparse")
    h = C.c_void_p()
    assert _native.lib().tfr_schema_create_ex(fields, 2, 0, A.TFR_S_RAGGED, C.byref(h)) == 0
    assert _native.lib().tfr_schema_num_fields(h) == 4               # sparse parts count, the lengths part does not
    _native.lib().tfr_schema_destroy(h)


@pytest.mark.parametrize("other", ["x_values", "x_row_lengths"])
def test_key_collisions_name_both_fields(other):
    s = StructType([StructField(other, LongType()), StructField("x", ArrayType(ArrayType(FloatType())))])
    rc, _, msg = _create(s)
    assert rc == A.TFR_E_INVALID_ARG and f"'{other}'" in msg and "'x'" in msg
    assert _create(s, flags=0)[0] == 0


def test_lowering_order_and_suffixes():
    low = RR.lowered_schema(X)
    assert [f.name for f in low.fields] == ["id", "x_values", "s_values", "x_row_lengths", "s_row_lengths"]
    assert [f.nullable for f in low.fields] == [False, True, False, True, True]
    assert RR.lower_row(X, (1, [[1, 2], [], [3]], [["a"]])) == (1, [1, 2, 3], ["a"], [2, 0, 1], [1])
    assert RR.lower_row(X, (1, None, [[]])) == (1, None, [], None, [0])
    assert RR.lower_row(X, (1, [], [])) == (1, [], [], [], [])


def test_lowered_bytes_parse_back_with_upb():
    data = RR.encode(X, [(7, [[1, 2], [], [3]], [["a", "b"], []])])
    ex = pyref.Example()
    ex.ParseFromString(data[12:-4])
    f = ex.features.feature
    assert set(f.keys()) == {"id", "x_values", "x_row_lengths", "s_values", "s_row_lengths"}
    assert list(f["x_values"].int64_list.value) == [1, 2, 3] and list(f["x_row_lengths"].int64_list.value) == [2, 0, 1]
    assert list(f["s_values"].bytes_list.value) == [b"a", b"b"] and list(f["s_row_lengths"].int64_list.value) == [2, 0]


def _payload(feats):
    return pyref.example(feats).SerializeToString()


def test_read_rules():
    i64, flt, byt = pyref.int64_feature, pyref.float_feature, pyref.bytes_feature
    base = {"id": i64(1), "s_values": byt(), "s_row_lengths": i64()}
    ok = dict(base, x_values=i64(1, 2, 3), x_row_lengths=i64(2, 0, 1))
    assert RR.read(X, _payload(ok)) == ((1, [[1, 2], [], [3]], []), None)
    assert RR.read(X, _payload(base)) == ((1, None, []), None)                         # both absent: null
    assert RR.read(X, _payload(dict(base, x_values=i64(1))))[1] == (A.TFR_E_BAD_NESTING, 1)
    assert RR.read(X, _payload(dict(base, x_row_lengths=i64(0))))[1] == (A.TFR_E_BAD_NESTING, 1)
    assert RR.read(X, _payload(dict(ok, x_row_lengths=i64(2, 2))))[1] == (A.TFR_E_BAD_NESTING, 1)
    assert RR.read(X, _payload(dict(ok, x_row_lengths=i64(4, -1, 0))))[1] == (A.TFR_E_BAD_NESTING, 1)
    assert RR.read(X, _payload(dict(ok, x_row_lengths=flt(1.0))))[1] == (A.TFR_E_KIND_MISMATCH, 1)
    # precedence: a caller field's error before the lengths part's, and that before the consistency check
    assert RR.read(X, _payload(dict(ok, id=flt(1.0), x_row_lengths=flt(1.0))))[1] == (A.TFR_E_KIND_MISMATCH, 0)
    bad_s = {"id": i64(1), "x_values": i64(1), "s_values": byt("a")}
    assert RR.read(X, _payload(bad_s))[1] == (A.TFR_E_BAD_NESTING, 1)                  # x (field 1) before s (field 2)
    assert RR.read(X, _payload({"id": i64(1)}))[1] == (A.TFR_E_NULL_IN_NONNULL, 2)     # non-nullable s absent


def test_jni_shim_maps_the_nested_array_format(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    assert "TfrGpu_schemaCreateFormat" in open(src).read()
    main = tmp_path / "m.cpp"
    main.write_text('#include "%s"\n#include <cstdio>\nint main() {\n'
                    '  const char* f[] = {"featureList", "ragged", "Ragged", ""};\n'
                    '  for (int rt = 0; rt < 3; ++rt) for (auto a : f) printf("%%lld ", (long long)nested_array_flags(a, rt));\n'
                    '  return 0;\n}\n' % src)
    exe = tmp_path / "m"
    p = subprocess.run(["g++", "-std=c++17", "-DTFR_BUILD_JNI", "-I", os.path.join(root, "tests", "jni_stub"), str(main), "-o", str(exe),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    #               Example              SequenceExample        ByteArray (ignores the flag)
    assert out == ["0", "1", "-1", "-1", "0", "-1", "-1", "-1", "0", "1", "-1", "-1"]
