"""BooleanType, ByteType, ShortType, DateType and TimestampType fields (include/tfrgpu.h, INT64 TYPES) restated on top of the
LongType oracle -- test infrastructure next to tests/ragged_rows.py.

With extendedTypes=true such a field IS a LongType field: a write is pyref's encoding of the LongType rows holding the widened
values, and a read is the oracle's LongType decode of the same bytes, narrowed in numpy.  UnsafeRows are restated from Spark's
UnsafeRowWriter / UnsafeArrayData: a scalar slot zeroed, then 1, 1, 2, 4 or 8 bytes; an array element 1, 1, 2, 4 or 8 bytes
wide, the element region rounded up to 8 bytes."""
from __future__ import annotations

import struct
from typing import List, Sequence

import numpy as np

from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import (ArrayType, BooleanType, ByteType, DateType, LongType, ShortType, StructField,
                                          StructType, TimestampType, lower_type)

# name -> (Spark type, tfr id, numpy dtype of the narrow leaf values, Arrow format)
TYPES = {
    "bool": (BooleanType(), A.TFR_T_BOOL, np.uint8, "b"),
    "byte": (ByteType(), A.TFR_T_INT8, np.int8, "c"),
    "short": (ShortType(), A.TFR_T_INT16, np.int16, "s"),
    "date": (DateType(), A.TFR_T_DATE, np.int32, "tdD"),
    "timestamp": (TimestampType(), A.TFR_T_TIMESTAMP, np.int64, "tsu:UTC"),
}
BY_ID = {v[1]: k for k, v in TYPES.items()}
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
# int64 values read back through every narrowing: a boolean that looks at the low 32 bits only fails on 2^32
EDGES = [0, 1, -1, 1 << 32, INT64_MIN, INT64_MAX, 300, -129, 70000, (1 << 32) + 5]


def _leaf(dt):
    while isinstance(dt, ArrayType):
        dt = dt.elementType
    return dt


def leaf_id(dt) -> int:
    """the INT64 TYPES id of a field's leaf type, 0 for any other type"""
    t, _ = lower_type(dt, extended_types=True)
    return t if t in A.INT64_TYPES else 0


def long_type(dt):
    if isinstance(dt, ArrayType):
        return ArrayType(long_type(dt.elementType))
    return LongType() if leaf_id(dt) else dt


def long_schema(schema: StructType) -> StructType:
    """the schema every kernel sees: each such leaf a LongType"""
    return StructType([StructField(f.name, long_type(f.dataType), f.nullable) for f in schema])


def widen(t: int, x: int) -> int:
    """a narrow leaf value (as its column holds it) -> the Int64 written"""
    return (1 if x else 0) if t == A.TFR_T_BOOL else int(x)


def narrow(t: int, v: np.ndarray) -> np.ndarray:
    """int64 leaf values -> the narrow leaf values a read gives"""
    v = np.asarray(v, dtype=np.int64)
    if t == A.TFR_T_BOOL:
        return (v != 0).astype(np.uint8)
    return v.astype(TYPES[BY_ID[t]][2])            # (numpy keeps the low bits: .toByte, .toShort, .toInt)


def _widen_value(t, v):
    if v is None:
        return None
    if isinstance(v, list):
        return [_widen_value(t, e) for e in v]
    return widen(t, v)


def long_rows(schema: StructType, rows: Sequence[Sequence]) -> List[tuple]:
    """rows of narrow leaf values (ints) -> the LongType rows of long_schema(schema)"""
    ids = [leaf_id(f.dataType) for f in schema]
    return [tuple(_widen_value(t, v) if t else v for t, v in zip(ids, row)) for row in rows]


def narrow_columns(schema: StructType, cols) -> list:
    """the oracle's LongType HostColumns of long_schema(schema) -> (elem_type, leaf values) per field as the read gives them"""
    out = []
    for f, c in zip(schema, cols):
        t = leaf_id(f.dataType)
        out.append((t, narrow(t, c.values)) if t else (c.elem_type, c.values))
    return out


# ---- UnsafeRows of a schema of LongType, FloatType and INT64 TYPES fields, from the narrow leaf values: what tfr_batch_rows
#      writes, and the input of tfr_encode_rows ----
def _width(t: int) -> int:
    return {A.TFR_T_BOOL: 1, A.TFR_T_INT8: 1, A.TFR_T_INT16: 2, A.TFR_T_DATE: 4}.get(t, 8)


def _elems(t: int, vals) -> bytes:
    w = _width(t)
    b = b"".join(int(v).to_bytes(w, "little", signed=w > 1 or t == A.TFR_T_INT8) if t != A.TFR_T_BOOL else bytes([int(v)])
                 for v in vals)
    return b + bytes(-len(b) % 8)


def unsafe_array(t: int, depth: int, v) -> bytes:
    n = len(v)
    head = struct.pack("<q", n) + bytes(8 * ((n + 63) // 64))
    if depth == 1:
        return head + _elems(t, v)
    slots, var = b"", b""
    base = len(head) + 8 * n
    for inner in v:
        a = unsafe_array(t, 1, inner)
        slots += struct.pack("<Q", ((base + len(var)) << 32) | len(a))
        var += a
    return head + slots + var


def unsafe_row(schema: StructType, row: Sequence) -> bytes:
    nf = len(schema.fields)
    nw = (nf + 63) // 64
    bits = [0] * nw
    slots, var = [], b""
    fixed = 8 * (nw + nf)
    for i, (f, v) in enumerate(zip(schema, row)):
        t, depth = lower_type(long_type(f.dataType)) if not leaf_id(f.dataType) else (leaf_id(f.dataType), 0)
        if leaf_id(f.dataType):
            depth = 0
            dt = f.dataType
            while isinstance(dt, ArrayType):
                depth += 1
                dt = dt.elementType
        if v is None:
            bits[i >> 6] |= 1 << (i & 63)
            slots.append(0)
        elif depth == 0 and t == A.TFR_T_FLOAT32:
            slots.append(struct.unpack("<I", struct.pack("<f", v))[0])
        elif depth == 0:
            w = _width(t)
            slots.append(int(v) & ((1 << (8 * w)) - 1))
        else:
            a = unsafe_array(t, depth, v)
            slots.append(((fixed + len(var)) << 32) | len(a))
            var += a
    return b"".join(struct.pack("<Q", x) for x in bits + slots) + var
