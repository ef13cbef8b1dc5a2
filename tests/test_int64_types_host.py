"""extendedTypes=true (include/tfrgpu.h, INT64 TYPES) without a GPU: the option and its refusals, the schema flag with and without
TFR_S_RAGGED, the new ids refused without it, the lowering, the Python value conversions, and the restatement in
tests/int64_types.py."""
import ctypes as C
import datetime as dt
import os
import subprocess

import numpy as np
import pytest

import int64_types as I
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native, io
from spark_tfrecord_b200.sqltypes import *  # noqa

ALL = StructType([StructField(n, t[0], True) for n, t in I.TYPES.items()] +
                 [StructField("a_" + n, ArrayType(t[0]), False) for n, t in I.TYPES.items()])


def _create(schema, rt=0, flags=A.TFR_S_INT64_TYPES, extended=True):
    fields, keep = A.make_fields(schema, extended_types=extended)
    h = C.c_void_p()
    rc = _native.lib().tfr_schema_create_ex(fields, len(schema), rt, flags, C.byref(h))
    n = _native.lib().tfr_schema_num_fields(h) if rc == 0 else None
    if rc == 0:
        _native.lib().tfr_schema_destroy(h)
    return rc, n, _native.lib().tfr_last_error().decode()


def test_option_values():
    assert io._extended_types({}) is False
    assert io._extended_types({"extendedTypes": "false"}) is False
    assert io._extended_types({"extendedTypes": "true"}) is True
    for bad in ("True", "1", "yes", ""):
        with pytest.raises(_native.IllegalArgumentException):
            io._extended_types({"extendedTypes": bad})
    with pytest.raises(_native.IllegalArgumentException):
        io.DefaultSource().prepareWrite({"extendedTypes": "on"}, ALL)
    with pytest.raises(_native.IllegalArgumentException):
        io.DefaultSource().buildReader(ALL, ALL, {"extendedTypes": "on"})
    with pytest.raises(_native.IllegalArgumentException):
        io.DefaultSource().inferSchema({"extendedTypes": "on"}, [])


def test_lowering():
    for n, (t, tid, _, _) in I.TYPES.items():
        assert lower_type(t) == (TFR_T_UNSUPPORTED, 0)                  # the reference's refusal without the option
        assert lower_type(t, extended_types=True) == (tid, 0)
        assert lower_type(ArrayType(ArrayType(t)), extended_types=True) == (tid, 2)
    assert lower_type(LongType(), extended_types=True) == (TFR_T_INT64, 0)
    assert I.long_schema(ALL).fields[7] == StructField("a_short", ArrayType(LongType()), False)


def test_schema_flag():
    rc, n, _ = _create(ALL)
    assert rc == 0 and n == len(ALL)
    for flags in (0, A.TFR_S_RAGGED):                                      # the new ids need the flag, naming the field
        rc, _, msg = _create(ALL, flags=flags)
        assert rc == A.TFR_E_UNSUPPORTED_TYPE and "'bool'" in msg
    nested = StructType([StructField("x", ArrayType(ArrayType(DateType())), True), StructField("b", BooleanType(), False)])
    assert _create(nested, 0, A.TFR_S_INT64_TYPES | A.TFR_S_RAGGED)[:2] == (0, 2)
    assert _create(nested, 1, A.TFR_S_INT64_TYPES)[:2] == (0, 2)          # SequenceExample FeatureLists
    assert _create(nested, 2, 0)[0] == 0                                   # a ByteArray schema ignores the types and the flag
    assert _create(nested, 0, 0x8)[0] == A.TFR_E_INVALID_ARG               # an unknown flag
    # with the option the Python schema sets the flag; without it the refusal is the reference's
    _native.Schema(ALL, 0, extended_types=True).close()
    with pytest.raises(_native.UnsupportedTypeException):
        _native.Schema(ALL, 0)


def test_python_values():
    utc = dt.timezone.utc
    cases = [(A.TFR_T_BOOL, True, 1), (A.TFR_T_BOOL, False, 0), (A.TFR_T_INT8, -128, -128), (A.TFR_T_INT16, 32767, 32767),
             (A.TFR_T_DATE, dt.date(1969, 12, 31), -1), (A.TFR_T_DATE, dt.date(2000, 3, 1), 11017),
             (A.TFR_T_TIMESTAMP, dt.datetime(1970, 1, 1, 0, 0, 0, 1, tzinfo=utc), 1),
             (A.TFR_T_TIMESTAMP, dt.datetime(1970, 1, 1, 1, 0, tzinfo=dt.timezone(dt.timedelta(hours=1))), 0)]
    for t, v, x in cases:
        assert A.int64_leaf(t, v) == x
        back = A.int64_value(t, x)
        assert back == v and (t != A.TFR_T_TIMESTAMP or back.tzinfo == utc)
    for t, v in [(A.TFR_T_INT8, 128), (A.TFR_T_INT8, -129), (A.TFR_T_INT16, 1 << 15), (A.TFR_T_TIMESTAMP, dt.datetime(2020, 1, 1)),
                 (A.TFR_T_DATE, "2020-01-01"), (A.TFR_T_BOOL, "yes"), (A.TFR_T_INT8, True)]:
        with pytest.raises(ValueError):
            A.int64_leaf(t, v)
    cols = A.columns_from_rows(ALL, [(True, -1, 2, dt.date(1970, 1, 2), dt.datetime(1970, 1, 1, tzinfo=utc), [False, True], [3],
                                      [-4], [dt.date(1970, 1, 1)], [])])
    assert [c.values.dtype for c in cols[:5]] == [np.uint8, np.int8, np.int16, np.int32, np.int64]
    assert [c.values.tolist() for c in cols] == [[1], [-1], [2], [1], [0], [0, 1], [3], [-4], [0], []]
    assert [c.get(0) for c in cols][:2] == [True, -1]


def test_restatement():
    # the narrowing keeps the low bits, a boolean looks at all 64
    v = np.array(I.EDGES, dtype=np.int64)
    assert I.narrow(A.TFR_T_BOOL, v).tolist() == [0, 1, 1, 1, 1, 1, 1, 1, 1, 1]
    assert I.narrow(A.TFR_T_INT8, v).tolist()[-4:] == [44, 127, 112, 5]
    assert I.narrow(A.TFR_T_INT16, v).tolist()[-2:] == [4464, 5]
    assert I.narrow(A.TFR_T_DATE, v).tolist()[2:4] == [-1, 0]
    # a written row is the LongType row with the widened values; upb reads it back as Int64 features
    sch = StructType([StructField("b", BooleanType(), True), StructField("d", ArrayType(DateType()), True)])
    [row] = I.long_rows(sch, [(1, [-1, 5])])
    ex = pyref.Example()
    ex.ParseFromString(pyref.serialize_example_bytes(I.long_schema(sch), row))
    assert list(ex.features.feature["b"].int64_list.value) == [1]
    assert list(ex.features.feature["d"].int64_list.value) == [-1, 5]
    # an UnsafeRow of a boolean and a short array: the slot's one byte, the 2-byte elements padded to 8
    r = I.unsafe_row(StructType([StructField("b", BooleanType(), True), StructField("s", ArrayType(ShortType()), True)]), [1, [-1, 2, 3]])
    assert r[:8] == bytes(8) and r[8:16] == (1).to_bytes(8, "little")
    assert r[16:24] == ((24 << 32) | 24).to_bytes(8, "little")
    assert r[24:] == (3).to_bytes(8, "little") + bytes(8) + b"\xff\xff\x02\x00\x03\x00\x00\x00"


def test_jni_shim_maps_the_extended_types(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    text = open(src).read()
    assert "TfrGpu_schemaCreateOptions" in text and "TfrGpu_extendedElemType" in text
    main = tmp_path / "m.cpp"
    main.write_text('#include "%s"\n#include <cstdio>\nint main() {\n'
                    '  const char* t[] = {"boolean", "byte", "short", "date", "timestamp", "long", "timestamp_ntz"};\n'
                    '  const char* v[] = {"true", "false", "TRUE"};\n'
                    '  for (auto o : v) for (auto n : t) printf("%%d ", extended_elem_type(n, o));\n'
                    '  for (auto o : v) printf("%%lld ", (long long)extended_types_flags(o));\n'
                    '  return 0;\n}\n' % src)
    exe = tmp_path / "m"
    p = subprocess.run(["g++", "-std=c++17", "-DTFR_BUILD_JNI", "-I", os.path.join(root, "tests", "jni_stub"), str(main), "-o", str(exe),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out[:7] == [A.TFR_T_BOOL, A.TFR_T_INT8, A.TFR_T_INT16, A.TFR_T_DATE, A.TFR_T_TIMESTAMP, -2, -2]   # "true"
    assert out[7:14] == [-1] * 5 + [-2, -2]                                                            # "false": refused
    assert out[14:21] == [-3] * 7                                                                      # another value
    assert out[21:] == [A.TFR_S_INT64_TYPES, 0, -1]
