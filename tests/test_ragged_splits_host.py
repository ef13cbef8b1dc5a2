"""raggedPartition=rowSplits (include/tfrgpu.h, RAGGED, Row splits) without a GPU: the option, the schema flag and its
refusals, the lowering, and the restatement in tests/ragged_splits_rows.py, whose bytes upb's tensorflow.Example parses back
into the two plain features."""
import ctypes as C
import os
import subprocess

import pytest

import ragged_splits_rows as RS
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native, io
from spark_tfrecord_b200.sqltypes import *  # noqa

X = StructType([StructField("id", LongType(), False), StructField("x", ArrayType(ArrayType(LongType())), True),
                StructField("s", ArrayType(ArrayType(StringType())), False)])
SPLITS = A.TFR_S_RAGGED | A.TFR_S_RAGGED_ROW_SPLITS


def _create(schema, rt=0, flags=SPLITS):
    fields, keep = A.make_fields(schema, extended_types=bool(flags & A.TFR_S_INT64_TYPES))
    h = C.c_void_p()
    rc = _native.lib().tfr_schema_create_ex(fields, len(schema), rt, flags, C.byref(h))
    n = _native.lib().tfr_schema_num_fields(h) if rc == 0 else None
    if rc == 0:
        _native.lib().tfr_schema_destroy(h)
    return rc, n, _native.lib().tfr_last_error().decode()


def test_option_values_and_refusals():
    assert io._ragged_partition({}) is False
    assert io._ragged_partition({"nestedArrayFormat": "ragged"}) is False
    assert io._ragged_partition({"nestedArrayFormat": "ragged", "raggedPartition": "rowLengths"}) is False
    assert io._ragged_partition({"nestedArrayFormat": "ragged", "raggedPartition": "rowSplits"}) is True
    assert io._ragged_partition({"raggedPartition": "rowLengths"}) is False
    for bad in ({"nestedArrayFormat": "ragged", "raggedPartition": "RowSplits"},
                {"nestedArrayFormat": "ragged", "raggedPartition": "valueRowIds"},
                {"raggedPartition": "rowSplits"},                                     # without nestedArrayFormat=ragged
                {"nestedArrayFormat": "featureList", "raggedPartition": "rowSplits"},
                {"nestedArrayFormat": "ragged", "raggedPartition": "rowSplits", "recordType": "SequenceExample"}):
        with pytest.raises(_native.IllegalArgumentException):
            io._ragged_partition(bad)
    opts = {"nestedArrayFormat": "ragged", "raggedPartition": "x"}
    with pytest.raises(_native.IllegalArgumentException):
        io.DefaultSource().prepareWrite(opts, X)
    with pytest.raises(_native.IllegalArgumentException):
        io.DefaultSource().buildReader(X, X, opts)
    with pytest.raises(_native.IllegalArgumentException):
        io.DefaultSource().buildReader(X, X, {"raggedPartition": "rowSplits"})


def test_schema_flags_and_counts():
    assert _create(X)[:2] == (0, 3)                                  # a ragged field stays one column
    rc, _, msg = _create(X, flags=A.TFR_S_RAGGED_ROW_SPLITS)         # alone: refused
    assert rc == A.TFR_E_INVALID_ARG and "ragged" in msg
    assert _create(X, flags=SPLITS | A.TFR_S_INT64_TYPES)[:2] == (0, 3)
    assert _create(X, flags=A.TFR_S_RAGGED_ROW_SPLITS | A.TFR_S_INT64_TYPES)[0] == A.TFR_E_INVALID_ARG
    assert _create(X, flags=SPLITS | 2)[0] == A.TFR_E_INVALID_ARG   # 0x2 stays an unknown flag
    rc, _, msg = _create(X, rt=1)
    assert rc == A.TFR_E_INVALID_ARG and "SequenceExample" in msg
    assert _create(X, rt=2)[0] == 0                                  # ByteArray ignores it
    b = StructType([StructField("x", ArrayType(ArrayType(BooleanType())), True)])
    assert _create(b, flags=SPLITS | A.TFR_S_INT64_TYPES)[:2] == (0, 1)
    sv = StructType([StructField("v", VectorUDT()), StructField("x", ArrayType(ArrayType(IntegerType())))])
    fields, keep = A.make_fields(sv, "sparse")
    h = C.c_void_p()
    assert _native.lib().tfr_schema_create_ex(fields, 2, 0, SPLITS, C.byref(h)) == 0
    assert _native.lib().tfr_schema_num_fields(h) == 4                # sparse parts count, the splits part does not
    _native.lib().tfr_schema_destroy(h)


@pytest.mark.parametrize("other", ["x_values", "x_row_splits"])
def test_key_collisions_name_both_fields(other):
    s = StructType([StructField(other, LongType()), StructField("x", ArrayType(ArrayType(FloatType())))])
    rc, _, msg = _create(s)
    assert rc == A.TFR_E_INVALID_ARG and f"'{other}'" in msg and "'x'" in msg
    assert _create(s, flags=0)[0] == 0


def test_lengths_key_does_not_collide_under_splits():
    s = StructType([StructField("x_row_lengths", LongType()), StructField("x", ArrayType(ArrayType(FloatType())))])
    assert _create(s)[0] == 0
    assert _create(s, flags=A.TFR_S_RAGGED)[0] == A.TFR_E_INVALID_ARG


def test_lowering_order_and_suffixes():
    low = RS.lowered_schema(X)
    assert [f.name for f in low.fields] == ["id", "x_values", "s_values", "x_row_splits", "s_row_splits"]
    assert [f.nullable for f in low.fields] == [False, True, False, True, True]
    assert RS.lower_row(X, (1, [[1, 2], [], [3]], [["a"]])) == (1, [1, 2, 3], ["a"], [0, 2, 2, 3], [0, 1])
    assert RS.lower_row(X, (1, None, [[]])) == (1, None, [], None, [0, 0])
    assert RS.lower_row(X, (1, [], [])) == (1, [], [], [0], [0])


def test_lowered_bytes_parse_back_with_upb():
    data = RS.encode(X, [(7, [[1, 2], [], [3]], [["a", "b"], []])])
    ex = pyref.Example()
    ex.ParseFromString(data[12:-4])
    f = ex.features.feature
    assert set(f.keys()) == {"id", "x_values", "x_row_splits", "s_values", "s_row_splits"}
    assert list(f["x_values"].int64_list.value) == [1, 2, 3] and list(f["x_row_splits"].int64_list.value) == [0, 2, 2, 3]
    assert list(f["s_values"].bytes_list.value) == [b"a", b"b"] and list(f["s_row_splits"].int64_list.value) == [0, 2, 2]


def _payload(feats):
    return pyref.example(feats).SerializeToString()


def test_read_rules():
    i64, flt, byt = pyref.int64_feature, pyref.float_feature, pyref.bytes_feature
    base = {"id": i64(1), "s_values": byt(), "s_row_splits": i64(0)}
    ok = dict(base, x_values=i64(1, 2, 3), x_row_splits=i64(0, 2, 2, 3))
    assert RS.read(X, _payload(ok)) == ((1, [[1, 2], [], [3]], []), None)
    assert RS.read(X, _payload(base)) == ((1, None, []), None)                          # both absent: null
    assert RS.read(X, _payload(dict(base, x_values=i64(), x_row_splits=i64(0)))) == ((1, [], []), None)
    assert RS.read(X, _payload(dict(base, x_values=i64(), x_row_splits=i64(0, 0)))) == ((1, [[]], []), None)
    for bad in (dict(base, x_values=i64(1)),                                             # exactly one part
                dict(base, x_row_splits=i64(0)),
                dict(ok, x_row_splits=i64()),                                            # an empty splits list
                dict(base, x_values=i64(), x_row_splits=i64()),
                dict(ok, x_row_splits=i64(1, 2, 3)),                                     # first entry not 0
                dict(ok, x_row_splits=i64(0, 3, 2, 3)),                                  # a decrease
                dict(ok, x_row_splits=i64(0, 2, 2, 4)),                                  # last entry not the values
                dict(ok, x_row_splits=i64(0, 2, 2))):
        assert RS.read(X, _payload(bad))[1] == (A.TFR_E_BAD_NESTING, 1)
    assert RS.read(X, _payload(dict(ok, x_row_splits=flt(0.0))))[1] == (A.TFR_E_KIND_MISMATCH, 1)
    # precedence: a caller field's error before the splits part's, and that before the consistency check
    assert RS.read(X, _payload(dict(ok, id=flt(1.0), x_row_splits=flt(1.0))))[1] == (A.TFR_E_KIND_MISMATCH, 0)
    assert RS.read(X, _payload(dict(ok, x_row_splits=flt(1.0), s_row_splits=i64(5))))[1] == (A.TFR_E_KIND_MISMATCH, 1)
    bad_s = {"id": i64(1), "x_values": i64(1), "s_values": byt("a")}
    assert RS.read(X, _payload(bad_s))[1] == (A.TFR_E_BAD_NESTING, 1)                   # x (field 1) before s (field 2)
    assert RS.read(X, _payload({"id": i64(1)}))[1] == (A.TFR_E_NULL_IN_NONNULL, 2)      # non-nullable s absent


def test_cross_partition_reads_fail():
    """a lengths file read with row splits and a splits file read with row lengths: x_values is there, the expected partition
    is not, so every record with x present is TFR_E_BAD_NESTING at x; neither partition is read as the other"""
    import ragged_rows as RR
    rows = [(1, [[1, 2], [3]], [["a"]]), (2, None, [])]
    lengths_payload = RR.encode(X, rows[:1])[12:-4]
    splits_payload = RS.encode(X, rows[:1])[12:-4]
    assert RS.read(X, lengths_payload)[1] == (A.TFR_E_BAD_NESTING, 1)
    assert RR.read(X, splits_payload)[1] == (A.TFR_E_BAD_NESTING, 1)
    assert RS.read(X, RR.encode(X, rows[1:])[12:-4])[1] == (A.TFR_E_BAD_NESTING, 2)     # x null, s's lengths without splits


def test_jni_shim_maps_the_ragged_partition(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    assert "TfrGpu_schemaCreatePartition" in open(src).read()
    main = tmp_path / "m.cpp"
    main.write_text('#include "%s"\n#include <cstdio>\nint main() {\n'
                    '  const char* f[] = {"featureList", "ragged"};\n'
                    '  const char* p[] = {"rowLengths", "rowSplits", "RowSplits", ""};\n'
                    '  for (int rt = 0; rt < 2; ++rt) for (auto a : f) for (auto b : p)\n'
                    '    printf("%%lld ", (long long)ragged_partition_flags(b, nested_array_flags(a, rt)));\n'
                    '  return 0;\n}\n' % src)
    exe = tmp_path / "m"
    p = subprocess.run(["g++", "-std=c++17", "-DTFR_BUILD_JNI", "-I", os.path.join(root, "tests", "jni_stub"), str(main), "-o", str(exe),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    #        Example: featureList        ragged               SequenceExample: featureList   ragged (refused)
    assert out == ["0", "-1", "-1", "-1", "0", "8", "-1", "-1", "0", "-1", "-1", "-1", "0", "-1", "-1", "-1"]
