"""Reads Spark UnsafeRows back into Python rows -- TEST INFRASTRUCTURE, independent of oracle.unsaferow's builder.

Parses the published UnsafeRow / UnsafeArrayData layout (include/tfrgpu.h): null bitset words, 8-byte slots, variable
values at (offset << 32) | size.  Checks the layout rules on the way (sizes and offsets in range, 8-byte alignment, zero
padding, element null bits clear) and raises ValueError naming what broke.  Values come back normalised for exact
comparison: fixed-width leaves as their bit patterns (ints), strings and binaries as bytes, arrays as lists, null as None."""
from __future__ import annotations

import struct
from typing import List, Sequence

import numpy as np

from spark_tfrecord_b200.sqltypes import (StructType, lower_type, TFR_T_NULL, TFR_T_INT32, TFR_T_FLOAT32, TFR_T_FLOAT64, TFR_T_STRING,
                                          TFR_T_BINARY)


def _u64(b: bytes, at: int) -> int:
    if at < 0 or at + 8 > len(b):
        raise ValueError(f"word at {at} outside {len(b)} bytes")
    return struct.unpack_from("<Q", b, at)[0]


def _var(b: bytes, slot: int, base: int, what: str) -> bytes:
    off, size = slot >> 32, slot & 0xFFFFFFFF
    if off % 8 or base + off + size > len(b):
        raise ValueError(f"{what}: offset {off} size {size} outside {len(b) - base} bytes or misaligned")
    pad = b[base + off + size:base + off + (size + 7) // 8 * 8]
    if any(pad):
        raise ValueError(f"{what}: non-zero padding")
    return b[base + off:base + off + size]


def _array(t: int, depth: int, b: bytes, what: str) -> list:
    n = struct.unpack_from("<q", b, 0)[0] if len(b) >= 8 else -1
    if n < 0:
        raise ValueError(f"{what}: bad numElements")
    nb = (n + 63) // 64 * 8
    if any(b[8:8 + nb]):
        raise ValueError(f"{what}: element null bit set")
    d = 8 + nb
    var = depth == 2 or t in (TFR_T_STRING, TFR_T_BINARY)
    if var:
        return [_array(t, 1, _var(b, _u64(b, d + 8 * i), 0, what), what) if depth == 2 else _var(b, _u64(b, d + 8 * i), 0, what)
                for i in range(n)]
    w = 4 if t in (TFR_T_INT32, TFR_T_FLOAT32) else 8
    if d + n * w > len(b) or any(b[d + n * w:d + (n * w + 7) // 8 * 8]):
        raise ValueError(f"{what}: elements outside the array or non-zero padding")
    return [int.from_bytes(b[d + i * w:d + (i + 1) * w], "little") for i in range(n)]


def read_row(schema: StructType, b: bytes) -> tuple:
    nf = len(schema)
    nw = (nf + 63) // 64
    if len(b) % 8 or len(b) < 8 * (nw + nf):
        raise ValueError(f"row of {len(b)} bytes")
    out = []
    for i, f in enumerate(schema):
        t, depth = lower_type(f.dataType)
        slot = _u64(b, 8 * (nw + i))
        if (_u64(b, 8 * (i >> 6)) >> (i & 63)) & 1:
            if slot:
                raise ValueError(f"field {i}: null with a non-zero slot")
            out.append(None)
            continue
        if t == TFR_T_NULL:
            raise ValueError(f"field {i}: NullType not null")
        if depth == 0 and t not in (TFR_T_STRING, TFR_T_BINARY):
            w = 4 if t in (TFR_T_INT32, TFR_T_FLOAT32) else 8
            if slot >> (8 * w):
                raise ValueError(f"field {i}: high bytes of a 4-byte slot set")
            out.append(slot)
            continue
        v = _var(b, slot, 0, f"field {i}")
        out.append(v if depth == 0 else _array(t, depth, v, f"field {i}"))
    return tuple(out)


def read_rows(schema: StructType, rows: np.ndarray, offs: Sequence[int]) -> List[tuple]:
    buf = np.asarray(rows, dtype=np.uint8).tobytes()
    return [read_row(schema, buf[int(offs[r]):int(offs[r + 1])]) for r in range(len(offs) - 1)]


def normalise(schema: StructType, row: Sequence) -> tuple:
    """a Python row (oracle.unsaferow's value conventions) in read_row's form"""
    def leaf(t, v):
        if isinstance(v, str):
            return v.encode("utf-8")
        if isinstance(v, (bytes, bytearray)):
            return bytes(v)
        w = 4 if t in (TFR_T_INT32, TFR_T_FLOAT32) else 8
        if t in (TFR_T_FLOAT32, TFR_T_FLOAT64):
            dt = np.float32 if w == 4 else np.float64
            return int(np.asarray(v, dtype=dt).view(np.uint32 if w == 4 else np.uint64))
        return int(v) & ((1 << (8 * w)) - 1)

    def val(t, depth, v):
        if v is None:
            return None
        if depth == 0:
            return leaf(t, v)
        return [val(t, depth - 1, x) for x in v]
    out = []
    for f, v in zip(schema, row):
        t, depth = lower_type(f.dataType)
        out.append(None if t == TFR_T_NULL else val(t, depth, v))
    return tuple(out)


def first_diff(schema: StructType, got_rows, got_offs, want_rows, want_offs) -> str:
    """where two row batches first differ: the row, then the field (for a failing assertion's message)"""
    got_offs, want_offs = np.asarray(got_offs, np.int64), np.asarray(want_offs, np.int64)
    if len(got_offs) != len(want_offs):
        return f"{len(got_offs) - 1} rows vs {len(want_offs) - 1}"
    g, w = np.asarray(got_rows, np.uint8).tobytes(), np.asarray(want_rows, np.uint8).tobytes()
    for r in range(len(got_offs) - 1):
        a, b = g[got_offs[r]:got_offs[r + 1]], w[want_offs[r]:want_offs[r + 1]]
        if a == b:
            continue
        try:
            ra, rb = read_row(schema, a), read_row(schema, b)
        except ValueError as e:
            return f"row {r}: {e}"
        for i, (x, y) in enumerate(zip(ra, rb)):
            if x != y:
                return f"row {r} field {i} ({schema[i].name}): {x!r} vs {y!r}"
        return f"row {r}: same values, different bytes ({len(a)} vs {len(b)})"
    return "rows equal, buffers differ" if g != w else "equal"
