"""CPU tests of the sparse-format VectorUDT field (include/tfrgpu.h, SPARSE VECTORS): the type id, the lowering and schema rules
of tfr_schema_create (depth, key collisions, the n + 2k counts), the `vectorFormat` option, the toSparse parts of dense and
sparse vectors, tests/sparse_vector_rows.py's nested rows against hand-written bytes, the JNI shim's mapping, and the lowered
Example bytes of oracle/pyref parsed back with upb's tensorflow.Example.  The kernels: test_gpu_sparse_vector.py."""
import math
import os
import re
import struct
import subprocess

import numpy as np
import pytest

import sparse_vector_rows as SV
import vector_rows as V
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import (ArrayType, DenseVector, DoubleType, IntegerType, LongType, SparseVector, StringType,
                                          StructField, StructType, TFR_T_SPARSE_VECTOR, TFR_T_VECTOR, VectorUDT, lower_type,
                                          lowered_schema, sparse_parts)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fields(*fs):
    return StructType([StructField(*f) for f in fs])


def n_fields(schema, vf="sparse", rt=0):
    s = _native.Schema(schema, rt, vf)
    try:
        return _native.lib().tfr_schema_num_fields(s.h)
    finally:
        s.close()


def test_enum_suffixes_and_lowering():
    h = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    assert re.search(r"TFR_T_SPARSE_VECTOR\s*=\s*11\b", h) and "SPARSE VECTORS:" in h
    for k, v in (("INDICES", "_indices"), ("VALUES", "_values"), ("SIZE", "_size")):
        assert re.search(rf'#define TFR_SPARSE_{k}_SUFFIX\s+"{v}"', h)
    assert TFR_T_SPARSE_VECTOR == 11 and A.TFR_T_SPARSE_VECTOR == 11
    assert lower_type(VectorUDT()) == (TFR_T_VECTOR, 0) and lower_type(VectorUDT(), "sparse") == (TFR_T_SPARSE_VECTOR, 0)
    sch = fields(("v", VectorUDT(), False), ("id", LongType()), ("w", VectorUDT()))
    low = lowered_schema(sch, "sparse")
    assert [(f.name, f.dataType, f.nullable) for f in low] == [
        ("v_values", ArrayType(DoubleType()), False), ("id", LongType(), True), ("w_values", ArrayType(DoubleType()), True),
        ("v_indices", ArrayType(IntegerType()), True), ("v_size", IntegerType(), True),
        ("w_indices", ArrayType(IntegerType()), True), ("w_size", IntegerType(), True)]
    assert [f.name for f in lowered_schema(sch)] == ["v", "id", "w"]


def test_schema_counts_and_depth():
    sch = fields(("id", LongType()), ("v", VectorUDT()), ("s", StringType()), ("w", VectorUDT(), False))
    assert n_fields(sch) == 4 + 4 and n_fields(sch, "dense") == 4
    for rt in (0, 1):
        assert n_fields(sch, rt=rt) == 8
        with pytest.raises(_native.TfrError) as e:
            _native.Schema(fields(("id", LongType()), ("vs", ArrayType(VectorUDT()))), rt, "sparse")
        assert e.value.code == A.TFR_E_UNSUPPORTED_TYPE and "'vs'" in str(e.value)
    assert n_fields(sch, rt=2) == 1                                   # a ByteArray schema ignores it


@pytest.mark.parametrize("other", ["v_values", "v_indices", "v_size"])
@pytest.mark.parametrize("first", [True, False], ids=["vector_first", "vector_second"])
def test_key_collisions(other, first):
    fs = [("v", VectorUDT()), (other, ArrayType(DoubleType()))]
    sch = fields(*(fs if first else fs[::-1]))
    with pytest.raises(_native.TfrError) as e:
        _native.Schema(sch, 0, "sparse")
    assert e.value.code == A.TFR_E_INVALID_ARG
    assert "'v'" in str(e.value) and f"'{other}'" in str(e.value), str(e.value)
    assert n_fields(sch, "dense") == 2                                  # no collision in the dense format
    # a sparse vector named a_values next to a: their keys (a_values_values, a_values, ...) do not collide
    assert n_fields(fields(("a", VectorUDT()), ("a_values", VectorUDT()))) == 6
    with pytest.raises(_native.TfrError) as e:
        _native.Schema(fields(("v", VectorUDT()), ("v", LongType())), 0, "sparse")
    assert e.value.code == A.TFR_E_INVALID_ARG and "duplicate" in str(e.value)


def test_vector_format_option_refused():
    for opts in ({"vectorFormat": "Sparse"}, {"vectorFormat": "csr"}, {"vectorFormat": ""}):
        with pytest.raises(_native.TfrError) as e:
            tio.DefaultSource().prepareWrite(opts, fields(("v", VectorUDT())))
        assert "vectorFormat" in str(e.value)
        with pytest.raises(_native.TfrError) as e:
            tio.DefaultSource().buildReader(fields(("v", VectorUDT())), fields(("v", VectorUDT())), opts)
        assert "vectorFormat" in str(e.value)
    with pytest.raises(ValueError, match="vectorFormat"):
        lower_type(VectorUDT(), "CSR")


def test_to_sparse_parts():
    d = DenseVector([0.0, -0.0, 1.5, float("nan"), 0.0, 1e-300, -2.0])
    idx, vals, size = sparse_parts(d)
    assert idx == [2, 3, 5, 6] and size == 7
    assert vals[0] == 1.5 and math.isnan(vals[1]) and vals[2] == 1e-300 and vals[3] == -2.0
    assert np.float32(vals[2]) == 0.0                                    # kept, then 0.0f through toFloat
    s = SparseVector(10, [1, 4, 7], [0.0, -0.0, 3.0])                  # stored zeros dropped
    assert sparse_parts(s) == ([7], [3.0], 10)
    assert sparse_parts(DenseVector(np.zeros(4))) == ([], [], 4)       # the zero vector
    assert sparse_parts(SparseVector(0, [], [])) == ([], [], 0)
    assert sparse_parts(None) == (None, None, None)
    cols = A.columns_from_rows(fields(("id", LongType()), ("v", VectorUDT())),
                               [(1, d), (2, None), (3, DenseVector([0.0]))], vector_format="sparse")
    assert len(cols) == 4
    assert cols[1].get(0)[0] == 1.5 and cols[1].get(1) is None and cols[1].get(2) == []
    assert cols[2].get(0) == [2, 3, 5, 6] and cols[2].get(1) is None and cols[2].get(2) == []
    assert cols[3].get(0) == 7 and cols[3].get(1) is None and cols[3].get(2) == 1


def _arr(n, esz, raw):
    return struct.pack("<q", n) + b"\0" * (8 * ((n + 63) // 64)) + raw + b"\0" * (-len(raw) % 8)


def test_sparse_nested_row_bytes():
    idx = _arr(2, 4, struct.pack("<2i", 1, 5))                           # 8 + 8 + 8 = 24 bytes
    val = _arr(2, 8, struct.pack("<2d", 2.0, -1.0))                      # 8 + 8 + 16 = 32 bytes
    want = struct.pack("<Q", 0) + struct.pack("<4Q", 0, 6, (40 << 32) | 24, (64 << 32) | 32) + idx + val
    assert SV.sparse_struct(6, [1, 5], [2.0, -1.0]) == want
    # a null size: bit 1 and a zero slot
    want = struct.pack("<Q", 2) + struct.pack("<4Q", 0, 0, (40 << 32) | 24, (64 << 32) | 32) + idx + val
    assert SV.sparse_struct(None, [1, 5], [2.0, -1.0]) == want
    # null indices: bit 2, a zero slot, and the values move up
    want = struct.pack("<Q", 4) + struct.pack("<4Q", 0, 6, 0, (40 << 32) | 32) + val
    assert SV.sparse_struct(6, None, [2.0, -1.0]) == want
    want = struct.pack("<Q", 6) + struct.pack("<4Q", 0, 0, 0, (40 << 32) | 8) + _arr(0, 8, b"")      # numElements only
    assert SV.sparse_struct(None, None, []) == want
    # in a row: (offset << 32) | size of the nested row
    sch = fields(("id", LongType()), ("v", VectorUDT()))
    rows, offs = SV.unsafe_rows(sch, [(7, SV.SparseParts(6, None, [2.0, -1.0]))])
    b = rows.tobytes()
    assert struct.unpack_from("<Q", b, 16)[0] == (24 << 32) | 72 and b[24:] == SV.sparse_struct(6, None, [2.0, -1.0])


def test_twin_rows():
    sch = fields(("v", VectorUDT()), ("id", LongType()), ("w", VectorUDT()))
    rows = [(SparseVector(5, [0, 3], [1.0, 0.0]), 1, None), (None, 2, DenseVector([0.0, 4.0]))]
    assert SV.twin_rows(sch, rows) == [([1.0], 1, None, [0], 5, None, None), (None, 2, [4.0], None, None, [1], 2)]


def test_jni_shim_maps_the_vector_format(tmp_path):
    src = os.path.join(ROOT, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    assert "TfrGpu_udtElemTypeFormat" in open(src).read()
    main = tmp_path / "m.cpp"
    main.write_text('#include "%s"\n#include <cstdio>\nint main() {\n'
                    '  const char* c[] = {"org.apache.spark.ml.linalg.VectorUDT", "org.apache.spark.mllib.linalg.VectorUDT", "x.Other"};\n'
                    '  const char* f[] = {"dense", "sparse", "Sparse"};\n'
                    '  for (auto a : c) for (auto b : f) printf("%%d ", udt_elem_type(a, b));\n  return 0;\n}\n' % src)
    exe = tmp_path / "m"
    p = subprocess.run(["g++", "-std=c++17", "-DTFR_BUILD_JNI", "-I", os.path.join(ROOT, "tests", "jni_stub"), str(main), "-o", str(exe),
                        "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert out == ["10", "11", "-2", "10", "11", "-2", "-1", "-1", "-2"]


def test_lowered_example_parses_with_upb():
    sch = fields(("id", LongType()), ("v", VectorUDT()), ("w", VectorUDT()))
    rows = [(1, SparseVector(2 ** 18, [3, 70000], [0.5, -2.0]), DenseVector([0.0, 0.0])), (2, None, DenseVector([1.0, -0.0, 3.0]))]
    tw = lowered_schema(sch, "sparse")
    for row, tr in zip(rows, SV.twin_rows(sch, rows)):
        ex = pyref.Example()
        ex.ParseFromString(pyref.serialize_example_bytes(tw, tr))
        feat = ex.features.feature
        if row[1] is None:
            assert set(feat) == {"id", "w_values", "w_indices", "w_size"}
        else:
            assert set(feat) == {"id", "v_values", "v_indices", "v_size", "w_values", "w_indices", "w_size"}
            assert feat["v_indices"].WhichOneof("kind") == "int64_list" and list(feat["v_indices"].int64_list.value) == [3, 70000]
            assert feat["v_values"].WhichOneof("kind") == "float_list" and list(feat["v_values"].float_list.value) == [0.5, -2.0]
            assert feat["v_size"].WhichOneof("kind") == "int64_list" and list(feat["v_size"].int64_list.value) == [2 ** 18]
        w = row[2].toSparse()
        assert list(feat["w_indices"].int64_list.value) == w.indices.tolist()
        assert list(feat["w_values"].float_list.value) == w.values.tolist()
        assert feat["w_values"].WhichOneof("kind") == "float_list"      # present, even when empty (the zero vector)
        assert list(feat["w_size"].int64_list.value) == [w.size]
