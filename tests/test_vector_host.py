"""CPU tests of the VectorUDT field (include/tfrgpu.h, VECTORS): the type id and its depth rules in tfr_schema_create, the
Python types and io.py's mapping, tests/vector_rows.py's struct bytes against hand-written layouts, SparseVector's checks
clause by clause, and the JNI shim's mapping by class name.  The kernels: test_gpu_vector.py."""
import os
import re
import struct
import subprocess

import numpy as np
import pytest

import vector_rows as V
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import (ArrayType, DenseVector, DoubleType, FloatType, LongType, SparseVector, StructField,
                                          StructType, TFR_T_FLOAT64, TFR_T_VECTOR, VectorUDT, lower_type)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fields(*fs):
    return StructType([StructField(*f) for f in fs])


def test_enum_in_header_and_bindings():
    h = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    assert re.search(r"TFR_T_VECTOR\s*=\s*10\b", h)
    assert "VECTORS:" in h and "NOT checked against a JVM" in h
    assert TFR_T_VECTOR == 10 and A.TFR_T_VECTOR == 10
    assert lower_type(VectorUDT()) == (TFR_T_VECTOR, 0)
    assert lower_type(ArrayType(VectorUDT())) == (TFR_T_VECTOR, 1)


def test_schema_depth_rules():
    ok = _native.Schema(fields(("id", LongType()), ("features", VectorUDT()), ("label", DoubleType(), False), ("v", VectorUDT(), False)))
    assert _native.lib().tfr_schema_num_fields(ok.h) == 4
    ok.close()
    for rt in (0, 1):
        for dt in (ArrayType(VectorUDT()), ArrayType(ArrayType(VectorUDT()))):
            with pytest.raises(_native.TfrError) as e:
                _native.Schema(fields(("id", LongType()), ("vs", dt)), rt)
            assert e.value.code == A.TFR_E_UNSUPPORTED_TYPE and "'vs'" in str(e.value), str(e.value)
    # a ByteArray schema ignores its data fields, vectors at any depth included
    ba = _native.Schema(fields(("vs", ArrayType(VectorUDT())), ("v", VectorUDT())), 2)
    assert _native.lib().tfr_schema_num_fields(ba.h) == 1
    ba.close()


def test_vector_values():
    d = DenseVector([1.5, -2.0, 0.0])
    assert d.size == 3 and d.toArray().dtype == np.float64 and d.toArray().tolist() == [1.5, -2.0, 0.0]
    s = SparseVector(5, [1, 3], [2.0, 4.0])
    assert s.toArray().tolist() == [0.0, 2.0, 0.0, 4.0, 0.0]
    assert s == DenseVector([0, 2, 0, 4, 0]) and DenseVector([0, 2, 0, 4, 0]) == s
    assert SparseVector(0, [], []).toArray().tolist() == [] and DenseVector([]).size == 0


@pytest.mark.parametrize("size,indices,values", [
    (-1, [], []),                       # size < 0
    (4, [0, 1], [1.0]),                 # indices and values of different lengths
    (4, [0], [1.0, 2.0]),
    (4, [4], [1.0]),                    # an index at size
    (4, [-1], [1.0]),                   # a negative index
    (4, [2, 1], [1.0, 2.0]),            # decreasing
    (4, [1, 1], [1.0, 2.0]),            # repeated
    (0, [0], [1.0]),                    # any index of a size-0 vector
])
def test_sparse_vector_checks(size, indices, values):
    with pytest.raises(ValueError):
        SparseVector(size, indices, values)


def test_columns_from_rows_takes_either_kind():
    sch = fields(("id", LongType()), ("v", VectorUDT()))
    rows = [(1, DenseVector([1.0, 2.5])), (2, SparseVector(4, [3], [7.0])), (3, None), (4, SparseVector(0, [], [])), (5, DenseVector([]))]
    got = A.columns_from_rows(sch, rows)
    want = A.columns_from_rows(V.as_double_schema(sch), V.as_double_rows(sch, rows))
    for g, w in zip(got, want):
        assert (g.elem_type, g.depth) == (w.elem_type, w.depth)
        assert np.array_equal(g.validity, w.validity) and all(np.array_equal(a, b) for a, b in zip(g.offsets, w.offsets))
        assert np.array_equal(g.values, w.values)
    assert got[1].elem_type == TFR_T_FLOAT64 and got[1].depth == 1
    assert got[1].offsets[0].tolist() == [0, 2, 6, 6, 6, 6]
    assert tio._row_bytes((1, SparseVector(1000, [1], [1.0]))) >= 8000


def test_io_reader_returns_dense_vectors():
    class _Col:
        def __init__(self, vals):
            self.vals = vals

        def get(self, r):
            return self.vals[r]

    class _Batch:
        n_rows = 2

        def to_host(self):
            return [_Col([1, 2]), _Col([[1.0, 2.0], None])]
    sch = fields(("id", LongType()), ("v", VectorUDT()))
    rows = tio._rows_of(_Batch(), sch)
    assert rows[0][0] == 1 and isinstance(rows[0][1], DenseVector) and rows[0][1].toArray().tolist() == [1.0, 2.0]
    assert rows[1][1] is None
    assert tio._rows_of(_Batch())[0][1] == [1.0, 2.0]          # ByteArray rows: no schema mapping


def _w(*ws):
    return struct.pack("<%dQ" % len(ws), *ws)


def test_struct_bytes_dense():
    got = V.vector_struct(DenseVector([1.5, -2.0]))
    arr = _w(2, 0) + struct.pack("<2d", 1.5, -2.0)
    assert got == _w(0b0110, 1, 0, 0, (40 << 32) | len(arr)) + arr
    assert V.vector_struct(DenseVector([])) == _w(0b0110, 1, 0, 0, (40 << 32) | 8) + _w(0)


def test_struct_bytes_sparse():
    got = V.vector_struct(SparseVector(5, [1, 3], [2.0, 4.0]))
    idx = _w(2, 0) + struct.pack("<2i", 1, 3)
    val = _w(2, 0) + struct.pack("<2d", 2.0, 4.0)
    assert got == _w(0, 0, 5, (40 << 32) | len(idx), ((40 + len(idx)) << 32) | len(val)) + idx + val
    odd = V.vector_struct(SparseVector(9, [8], [1.0]))              # 4 bytes of indices pad to 8
    assert odd[40:40 + 24] == _w(1, 0) + struct.pack("<i", 8) + b"\0" * 4
    # size 0: empty arrays
    assert V.vector_struct(SparseVector(0, [], [])) == _w(0, 0, 0, (40 << 32) | 8, (48 << 32) | 8) + _w(0) + _w(0)


def test_struct_in_row_and_null():
    sch = fields(("id", LongType()), ("v", VectorUDT()))
    st = V.vector_struct(DenseVector([3.0]))
    row = V.unsafe_row(sch, (7, DenseVector([3.0])))
    assert row == _w(0, 7, (24 << 32) | len(st)) + st
    assert V.unsafe_row(sch, (7, None)) == _w(0b10, 7, 0)


def test_jni_shim_maps_the_udt_by_class_name():
    src = os.path.join(ROOT, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    text = open(src).read()
    assert "TfrGpu_udtElemType" in text
    for name in VectorUDT.CLASS_NAMES:
        assert f'"{name}"' in text
    p = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-DTFR_BUILD_JNI", "-I", os.path.join(ROOT, "tests", "jni_stub"), src],
                       capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr
