"""Spark UnsafeRow bytes from Python rows -- TEST/BENCH INFRASTRUCTURE for tfr_encode_rows.

Restates what Spark's UnsafeRowWriter / UnsafeArrayWriter produce (the published UnsafeRow / UnsafeArrayData format, see
include/tfrgpu.h): a null bitset of 64-bit words, one 8-byte slot per field, then the variable-length region, every
variable-length value starting on an 8-byte boundary with zeroed padding.  A null field has its bit set and a zero slot;
a null array element has its bit set and a zeroed element slot, or -- with `garbage=True` -- random bits in the slots of
null numeric elements (the encoder must copy them, like toIntArray / toFloatArray do); NullElem(v) is a null numeric
element whose slot holds v's bits.

Values follow columns_from_rows: int, float, str, bytes, list, list of lists, None; DecimalType takes the unscaled int64.
The product package never imports this module."""
from __future__ import annotations

import struct
from typing import List, Sequence, Tuple

import numpy as np

from spark_tfrecord_b200.sqltypes import (StructType, lower_type, TFR_T_NULL, TFR_T_INT32, TFR_T_INT64, TFR_T_FLOAT32,
                                          TFR_T_FLOAT64, TFR_T_DECIMAL, TFR_T_STRING, TFR_T_BINARY)

_ELEM_SIZE = {TFR_T_INT32: 4, TFR_T_FLOAT32: 4, TFR_T_INT64: 8, TFR_T_FLOAT64: 8, TFR_T_DECIMAL: 8}


class NullElem:
    """a null array element whose slot holds `value`'s bits (Spark writes 0 there: NullElem(0)); for numeric arrays only"""

    def __init__(self, value=0):
        self.value = value


def _pad8(b: bytes) -> bytes:
    return b + b"\0" * (-len(b) % 8)


def _scalar_bits(t: int, v) -> int:
    """the 64-bit slot of a fixed-width value (numpy float scalars keep their exact bits, NaN payloads included)"""
    if isinstance(v, np.floating):
        return int(np.asarray(v).view(np.uint32 if v.dtype == np.float32 else np.uint64))
    if t == TFR_T_INT32:
        return int(v) & 0xFFFFFFFF
    if t == TFR_T_FLOAT32:
        return struct.unpack("<I", struct.pack("<f", float(v)))[0]
    if t == TFR_T_FLOAT64:
        return struct.unpack("<Q", struct.pack("<d", float(v)))[0]
    return int(v) & 0xFFFFFFFFFFFFFFFF                                   # LongType, DecimalType (unscaled)


def _leaf_bytes(t: int, v) -> bytes:
    return v.encode("utf-8") if isinstance(v, str) else bytes(v)


def unsafe_array(t: int, depth: int, values: Sequence, rng=None) -> bytes:
    """UnsafeArrayData of `values`: depth 1 = array<leaf>, depth 2 = array<array<leaf>>"""
    n = len(values)
    nulls = bytearray(8 * ((n + 63) // 64))
    var_elem = depth == 2 or t in (TFR_T_STRING, TFR_T_BINARY)
    esz = 8 if var_elem else _ELEM_SIZE[t]
    header = 8 + len(nulls)
    fixed = bytearray(((n * esz) + 7) // 8 * 8)
    tail = bytearray()
    for i, v in enumerate(values):
        if isinstance(v, NullElem):
            nulls[i >> 3] |= 1 << (i & 7)
            fixed[i * esz:(i + 1) * esz] = _scalar_bits(t, v.value).to_bytes(8, "little")[:esz]
            continue
        if v is None:
            nulls[i >> 3] |= 1 << (i & 7)
            if rng is not None and not var_elem:
                fixed[i * esz:(i + 1) * esz] = rng.integers(1, 256, esz, dtype=np.uint8).tobytes()
            continue
        if var_elem:
            data = unsafe_array(t, 1, v, rng) if depth == 2 else _leaf_bytes(t, v)
            off = header + len(fixed) + len(tail)
            fixed[i * 8:(i + 1) * 8] = struct.pack("<Q", (off << 32) | len(data))
            tail += _pad8(data)
        else:
            fixed[i * esz:(i + 1) * esz] = _scalar_bits(t, v).to_bytes(8, "little")[:esz]
    return struct.pack("<q", n) + bytes(nulls) + bytes(fixed) + bytes(tail)


def unsafe_row(schema: StructType, row: Sequence, garbage: bool = False, seed: int = 0) -> bytes:
    """one UnsafeRow; garbage=True puts random bits in the slots of null numeric array elements"""
    rng = np.random.default_rng(seed) if garbage else None
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
        if depth == 0 and t not in (TFR_T_STRING, TFR_T_BINARY):
            slots[8 * i:8 * i + 8] = struct.pack("<Q", _scalar_bits(t, v))
            continue
        data = _leaf_bytes(t, v) if depth == 0 else unsafe_array(t, depth, v, rng)
        slots[8 * i:8 * i + 8] = struct.pack("<Q", ((head + len(tail)) << 32) | len(data))
        tail += _pad8(data)
    return bytes(nulls) + bytes(slots) + bytes(tail)


def unsafe_rows(schema: StructType, rows: Sequence[Sequence], garbage: bool = False, seed: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """-> (row bytes as uint8, int32 offsets[n + 1]), rows back to back"""
    parts: List[bytes] = [unsafe_row(schema, r, garbage, seed + k) for k, r in enumerate(rows)]
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(p) for p in parts])
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), offs.astype(np.int32)


def cfg2_rows(cols, n_int=32, n_float=16, n_bytes=16, float_len=8, bytes_len=16) -> Tuple[np.ndarray, np.ndarray]:
    """vectorised UnsafeRows of oracle.corpus.cfg2_columns (no nulls): n_int longs, n_float float[float_len] arrays,
    n_bytes binaries of bytes_len bytes.  -> (uint8 rows, int32 offsets)"""
    nf = n_int + n_float + n_bytes
    n = cols[0].n_rows
    nw = (nf + 63) // 64
    arr_bytes = 8 + 8 * ((float_len + 63) // 64) + (4 * float_len + 7) // 8 * 8
    bin_bytes = (bytes_len + 7) // 8 * 8
    head = 8 * (nw + nf)
    size = head + n_float * arr_bytes + n_bytes * bin_bytes
    R = np.zeros((n, size), dtype=np.uint8)
    slots = R[:, 8 * nw:head].view(np.uint64)
    for i in range(n_int):
        slots[:, i] = cols[i].values.view(np.uint64)
    for k in range(n_float):
        off = head + k * arr_bytes
        slots[:, n_int + k] = np.uint64((off << 32) | arr_bytes)
        R[:, off:off + 8].view(np.int64)[:, 0] = float_len
        v0 = off + arr_bytes - (4 * float_len + 7) // 8 * 8
        R[:, v0:v0 + 4 * float_len] = cols[n_int + k].values.reshape(n, float_len).view(np.uint8).reshape(n, 4 * float_len)
    for k in range(n_bytes):
        off = head + n_float * arr_bytes + k * bin_bytes
        slots[:, n_int + n_float + k] = np.uint64((off << 32) | bytes_len)
        R[:, off:off + bytes_len] = cols[n_int + n_float + k].values.reshape(n, bytes_len)
    offs = (np.arange(n + 1, dtype=np.int64) * size).astype(np.int32)
    return R.reshape(-1), offs
