"""VectorUDT values as Spark UnsafeRow bytes and the vector rules of the reference -- test infrastructure for the VectorUDT
field (include/tfrgpu.h, VECTORS), next to oracle/unsaferow.py and oracle/pyref.py, whose other rules it reuses.

A VectorUDT value is what UnsafeProjection makes of VectorUDT.serialize(v): the 8-byte slot (offset << 32) | size of a nested
UnsafeRow struct<type: tinyint, size: int, indices: array<int>, values: array<double>> -- one null word, four slots, then
the indices and values arrays in field order, each 8-byte aligned, offsets relative to the nested row:
  DenseVector : type 1, size and indices null (bits 1 and 2, zero slots), values.
  SparseVector: type 0, size, indices, values.
On write a vector is ArrayType(DoubleType) of v.toArray (pyref's DoubleType rule: each value through toFloat); on read it is
the ArrayType(DoubleType) column of the same field, as a dense vector."""
from __future__ import annotations

import struct
from typing import List, Optional, Sequence, Tuple

import numpy as np

from oracle.unsaferow import _leaf_bytes, _pad8, _scalar_bits, unsafe_array
from spark_tfrecord_b200.sqltypes import (ArrayType, DenseVector, DoubleType, SparseVector, StructField, StructType, VectorUDT,
                                          TFR_T_NULL, TFR_T_STRING, TFR_T_BINARY, lower_type)


def _array(raw: bytes, n: int, esz: int) -> bytes:
    """UnsafeArrayData of n elements of esz bytes given as raw little-endian bytes, no null element"""
    return struct.pack("<q", n) + b"\0" * (8 * ((n + 63) // 64)) + _pad8(raw)


def double_array(values) -> bytes:
    v = np.ascontiguousarray(values, dtype=np.float64)
    return _array(v.tobytes(), len(v), 8)


def int_array(values) -> bytes:
    v = np.ascontiguousarray(values, dtype=np.int32)
    return _array(v.tobytes(), len(v), 4)


def struct_bytes(type_byte: int, size: Optional[int], indices: Optional[bytes], values: Optional[bytes],
                 type_null: bool = False) -> bytes:
    """the nested row from its parts: `indices` / `values` are UnsafeArrayData bytes or None (null); size None: null"""
    nulls = (1 if type_null else 0) | (2 if size is None else 0) | (4 if indices is None else 0) | (8 if values is None else 0)
    slots = [type_byte & 0xFF, 0 if size is None else size & 0xFFFFFFFF, 0, 0]
    tail = b""
    for k, arr in ((2, indices), (3, values)):
        if arr is not None:
            slots[k] = ((40 + len(tail)) << 32) | len(arr)
            tail += _pad8(arr)
    return struct.pack("<Q", nulls) + struct.pack("<4Q", *slots) + tail


def vector_struct(v) -> bytes:
    """VectorUDT.serialize(v) as UnsafeProjection writes it"""
    if isinstance(v, SparseVector):
        return struct_bytes(0, v.size, int_array(v.indices), double_array(v.values))
    if not isinstance(v, DenseVector):
        v = DenseVector(v)
    return struct_bytes(1, None, None, double_array(v.values))


class RawVector:
    """a vector field given as the nested row's bytes as they are (malformed structs), and the slot's size (default: all)"""

    def __init__(self, data: bytes, size: Optional[int] = None, offset_delta: int = 0):
        self.data, self.size, self.offset_delta = data, size, offset_delta


def unsafe_row(schema: StructType, row: Sequence) -> bytes:
    """oracle.unsaferow.unsafe_row, with VectorUDT fields (DenseVector, SparseVector or RawVector values)"""
    nf = len(schema)
    nulls = bytearray(8 * ((nf + 63) // 64))
    slots = bytearray(8 * nf)
    head = len(nulls) + len(slots)
    tail = bytearray()
    for i, f in enumerate(schema):
        t, depth = lower_type(f.dataType)
        v = row[i]
        if v is None or t == TFR_T_NULL:
            nulls[i >> 3] |= 1 << (i & 7)
            continue
        if isinstance(f.dataType, VectorUDT):
            raw = v if isinstance(v, RawVector) else RawVector(vector_struct(v))
            size = len(raw.data) if raw.size is None else raw.size
            slots[8 * i:8 * i + 8] = struct.pack("<Q", ((head + len(tail) + raw.offset_delta) << 32) | size)
            tail += _pad8(raw.data)
            continue
        if depth == 0 and t not in (TFR_T_STRING, TFR_T_BINARY):
            slots[8 * i:8 * i + 8] = struct.pack("<Q", _scalar_bits(t, v))
            continue
        data = _leaf_bytes(t, v) if depth == 0 else unsafe_array(t, depth, v)
        slots[8 * i:8 * i + 8] = struct.pack("<Q", ((head + len(tail)) << 32) | len(data))
        tail += _pad8(data)
    return bytes(nulls) + bytes(slots) + bytes(tail)


def unsafe_rows(schema: StructType, rows: Sequence[Sequence]) -> Tuple[np.ndarray, np.ndarray]:
    """-> (row bytes as uint8, int32 offsets[n + 1]), rows back to back"""
    parts: List[bytes] = [unsafe_row(schema, r) for r in rows]
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(p) for p in parts])
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), offs.astype(np.int32)


def as_double_schema(schema: StructType) -> StructType:
    """the schema with every VectorUDT field as ArrayType(DoubleType) of the same name and nullability"""
    return StructType([StructField(f.name, ArrayType(DoubleType()), f.nullable) if isinstance(f.dataType, VectorUDT) else f
                       for f in schema])


def as_double_rows(schema: StructType, rows: Sequence[Sequence]) -> List[tuple]:
    """the rows with every vector as the list of its toArray: what the vector field writes"""
    out = []
    for row in rows:
        out.append(tuple(v.toArray().tolist() if isinstance(f.dataType, VectorUDT) and v is not None else v
                         for f, v in zip(schema, row)))
    return out
