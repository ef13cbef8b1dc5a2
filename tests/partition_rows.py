"""Spark UnsafeRows of D ++ P -- a data row joined with a file's partition values -- from values.  TEST INFRASTRUCTURE for
tfr_batch_rows_with_partition.

Restates what GenerateUnsafeProjection over D ++ P writes for JoinedRow(dataRow, partitionValues), through Spark's
UnsafeRowWriter: one null bitset of (nd + np + 63) / 64 words, nd + np slots, then the variable values in field order (the
data fields' as oracle.unsaferow writes them, then the partition fields'), each 8-byte aligned with zeroed padding.
Partition fields take their own type descriptors: "boolean", "byte", "short", "int", "long", "float", "double", "date"
(int days), "timestamp" (long microseconds), "string", "binary", ("decimal", precision, scale) with the unscaled int as
the value.  The rows are built field by field from the values, never by joining row bytes, so they check the GPU's
relocation of the partition row independently.  The same writer over P alone (nd = 0) gives the input partition row."""
from __future__ import annotations

import struct
from typing import List, Sequence, Tuple

import numpy as np

from oracle import unsaferow as U
from spark_tfrecord_b200.sqltypes import StructType, lower_type, TFR_T_NULL, TFR_T_STRING, TFR_T_BINARY

PART_TYPES = ["boolean", "byte", "short", "int", "long", "float", "double", "date", "timestamp", "string", "binary",
              ("decimal", 10, 2), ("decimal", 38, 6)]

_FIXED = {"boolean": "<?", "byte": "<b", "short": "<h", "int": "<i", "date": "<i", "long": "<q", "timestamp": "<q",
          "float": "<f", "double": "<d"}


def is_var(t) -> bool:
    """the slot is (offset << 32) | size: StringType, BinaryType, DecimalType with precision > 18"""
    return t in ("string", "binary") or (isinstance(t, tuple) and t[1] > 18)


def var_flags(ptypes) -> bytes:
    return bytes(1 if is_var(t) else 0 for t in ptypes)


def big_decimal_bytes(unscaled: int) -> bytes:
    """java.math.BigInteger.toByteArray(): big-endian, minimal two's complement (at least one byte)"""
    bits = unscaled.bit_length() if unscaled >= 0 else (-unscaled - 1).bit_length()
    return unscaled.to_bytes(bits // 8 + 1, "big", signed=True)


class _Writer:
    def __init__(self, n_fields: int):
        self.nulls = bytearray(8 * ((n_fields + 63) // 64))
        self.slots = bytearray(8 * n_fields)
        self.tail = bytearray()

    def cursor(self) -> int:
        return len(self.nulls) + len(self.slots) + len(self.tail)

    def set_null(self, i: int):
        self.nulls[i >> 3] |= 1 << (i & 7)
        self.slots[8 * i:8 * i + 8] = bytes(8)                # setNullAt zeroes the slot

    def slot(self, i: int, word: int):
        self.slots[8 * i:8 * i + 8] = struct.pack("<Q", word & 0xFFFFFFFFFFFFFFFF)

    def var(self, i: int, data: bytes):
        self.slot(i, (self.cursor() << 32) | len(data))
        self.tail += U._pad8(data)

    def row(self) -> bytes:
        return bytes(self.nulls) + bytes(self.slots) + bytes(self.tail)


def _write_partition(w: _Writer, k: int, t, v):
    if isinstance(t, tuple):                                 # ("decimal", precision, scale), v the unscaled int
        if t[1] <= 18:
            if v is None:
                w.set_null(k)
            else:
                w.slot(k, v)
            return
        off = w.cursor()                                     # 16 zeroed bytes, reserved for null values too
        w.tail += bytes(16)
        if v is None:
            w.nulls[k >> 3] |= 1 << (k & 7)
            w.slot(k, off << 32)
        else:
            b = big_decimal_bytes(v)
            assert len(b) <= 16
            start = len(w.tail) - 16                         # the bytes at the start of the reserved 16
            w.tail[start:start + len(b)] = b
            w.slot(k, (off << 32) | len(b))
        return
    if v is None:
        w.set_null(k)
    elif t == "string":
        w.var(k, v.encode("utf-8"))
    elif t == "binary":
        w.var(k, bytes(v))
    else:                                                    # the slot is zeroed, then 1, 2, 4 or 8 bytes written
        b = struct.pack(_FIXED[t], v)
        w.slot(k, int.from_bytes(b + bytes(8 - len(b)), "little"))


def write_data_field(w: _Writer, i: int, f, v):
    """data field i of value v, as oracle.unsaferow.unsafe_row writes it"""
    t, depth = lower_type(f.dataType)
    if v is None or t == TFR_T_NULL:
        w.set_null(i)
    elif depth == 0 and t not in (TFR_T_STRING, TFR_T_BINARY):
        w.slot(i, U._scalar_bits(t, v))
    else:
        w.var(i, U._leaf_bytes(t, v) if depth == 0 else U.unsafe_array(t, depth, v))


def joined_row(data_schema: StructType, data_row: Sequence, ptypes: Sequence, pvalues: Sequence,
               write_field=write_data_field) -> bytes:
    """`write_field(w, i, field, value)` writes one data field (tests/composed_rows.py passes the one of its lowerings)"""
    nd = len(data_schema)
    w = _Writer(nd + len(ptypes))
    for i, f in enumerate(data_schema):
        write_field(w, i, f, data_row[i])
    for j, (t, v) in enumerate(zip(ptypes, pvalues)):
        _write_partition(w, nd + j, t, v)
    return w.row()


def partition_row(ptypes: Sequence, pvalues: Sequence) -> bytes:
    """the UnsafeRow of the partition schema alone: what the caller passes"""
    return joined_row(StructType([]), [], ptypes, pvalues)


def joined_rows(data_schema: StructType, rows: Sequence[Sequence], ptypes, pvalues,
                write_field=write_data_field) -> Tuple[np.ndarray, np.ndarray]:
    """-> (row bytes as uint8, int64 offsets[n + 1]), rows back to back"""
    parts: List[bytes] = [joined_row(data_schema, r, ptypes, pvalues, write_field) for r in rows]
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(p) for p in parts])
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy(), offs


def cfg2_joined_rows(cols, ptypes, pvalues, n_int=32, n_float=16, n_bytes=16, float_len=8, bytes_len=16):
    """vectorised joined rows of oracle.corpus.cfg2_columns (no nulls, every row the same size).  The data part follows
    oracle.unsaferow.cfg2_rows with the larger fixed region; the partition part is written by the writer above into the
    first row's place and repeated.  Tests check it against joined_rows on a prefix.  -> (uint8 rows, int64 offsets)"""
    nd = n_int + n_float + n_bytes
    n = cols[0].n_rows
    nf = nd + len(ptypes)
    nw = (nf + 63) // 64
    arr_bytes = 8 + 8 * ((float_len + 63) // 64) + (4 * float_len + 7) // 8 * 8
    bin_bytes = (bytes_len + 7) // 8 * 8
    head = 8 * (nw + nf)
    dsize = head + n_float * arr_bytes + n_bytes * bin_bytes
    # the partition fields' slots, null bits and variable values as the writer lays them out behind this data part
    w = _Writer(nf)
    w.tail = bytearray(dsize - head)
    for j, (t, v) in enumerate(zip(ptypes, pvalues)):
        _write_partition(w, nd + j, t, v)
    prow = np.frombuffer(w.row(), np.uint8)
    size = len(prow)
    R = np.zeros((n, size), dtype=np.uint8)
    R[:, :8 * nw] = prow[:8 * nw]
    R[:, 8 * (nw + nd):head] = prow[8 * (nw + nd):head]
    R[:, dsize:] = prow[dsize:]
    slots = R[:, 8 * nw:8 * (nw + nd)].view(np.uint64)
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
    return R.reshape(-1), np.arange(n + 1, dtype=np.int64) * size
