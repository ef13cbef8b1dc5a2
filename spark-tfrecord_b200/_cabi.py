"""ctypes mirror of include/tfrgpu.h (struct layouts, status codes, column <-> numpy helpers).

Pure Python, no native code is loaded here; `_native.py` loads libtfrgpu.so."""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence

import numpy as np

from .sqltypes import (StructType, lower_type, TFR_T_NULL, TFR_T_INT32, TFR_T_INT64, TFR_T_FLOAT32,
                       TFR_T_FLOAT64, TFR_T_DECIMAL, TFR_T_STRING, TFR_T_BINARY, TFR_T_ROW_INDEX, TFR_T_RECORD_OFFSET,
                       TFR_T_VECTOR, TFR_T_SPARSE_VECTOR, lowered_schema, sparse_parts, sparse_vector_fields,
                       TFR_T_BOOL, TFR_T_INT8, TFR_T_INT16, TFR_T_DATE, TFR_T_TIMESTAMP, INT64_TYPES, int64_leaf, int64_value)

TFR_OK = 0
TFR_E_INVALID_ARG = -1
TFR_E_UNSUPPORTED_TYPE = -2
TFR_E_BAD_RECORD_TYPE = -3
TFR_E_CUDA = -4
TFR_E_OOM = -5
TFR_E_BATCH_TOO_LARGE = -6
TFR_E_CRC_LENGTH = -10
TFR_E_CRC_DATA = -11
TFR_E_TRUNCATED = -12
TFR_E_RECORD_TOO_LARGE = -13
TFR_E_MALFORMED_PROTO = -14
TFR_E_KIND_MISMATCH = -15
TFR_E_EMPTY_SCALAR = -16
TFR_E_NULL_IN_NONNULL = -17
TFR_E_BAD_NESTING = -18
TFR_E_INDEX_MISMATCH = -19     # a record index that does not describe its file (include/tfrgpu.h, RECORD INDEX)

TFR_F_VERIFY_CRC = 0x1
TFR_F_DROP_MALFORMED = 0x2       # mode=DROPMALFORMED: failing records are dropped, framing errors still end the block
TFR_F_PERMISSIVE = 0x4           # mode=PERMISSIVE: a failing record is a row of nulls (its payload in the corrupt-record column)
TFR_F_RESYNC = 0x8               # with DROPMALFORMED or PERMISSIVE: a framing error is a lost region, framing goes on at the next verified frame
TFR_F_DEFAULT = TFR_F_VERIFY_CRC

# the record errors a TFR_F_DROP_MALFORMED decoder drops (the other data errors are framing errors)
RECORD_ERRORS = (TFR_E_CRC_DATA, TFR_E_MALFORMED_PROTO, TFR_E_KIND_MISMATCH, TFR_E_EMPTY_SCALAR, TFR_E_NULL_IN_NONNULL,
                 TFR_E_BAD_NESTING)

# the framing errors: under TFR_F_RESYNC each names a lost region in tfr_batch_dropped / tfr_infer_skipped
FRAMING_ERRORS = (TFR_E_CRC_LENGTH, TFR_E_TRUNCATED, TFR_E_RECORD_TOO_LARGE)

STATUS_NAMES = {v: k for k, v in list(globals().items()) if k.startswith("TFR_E_") or k == "TFR_OK"}


class tfr_field(C.Structure):
    _fields_ = [("name", C.c_char_p), ("name_len", C.c_int32), ("elem_type", C.c_int32),
                ("depth", C.c_int32), ("nullable", C.c_int32)]


class tfr_batch_info(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_records", C.c_int64), ("consumed_bytes", C.c_int64),
                ("error_code", C.c_int32), ("error_row", C.c_int64), ("error_field", C.c_int32),
                ("out_bytes", C.c_int64), ("frame_repairs", C.c_int32)]


class tfr_column(C.Structure):
    _fields_ = [("elem_type", C.c_int32), ("depth", C.c_int32), ("n_levels", C.c_int32),
                ("value_width", C.c_int32), ("n_rows", C.c_int64), ("null_count", C.c_int64),
                ("validity", C.c_void_p), ("offsets", C.c_void_p * 3), ("n_offsets", C.c_int64 * 3),
                ("values", C.c_void_p), ("n_values", C.c_int64)]


_LEAF_DTYPE = {TFR_T_INT32: np.int32, TFR_T_INT64: np.int64, TFR_T_FLOAT32: np.float32,
               TFR_T_FLOAT64: np.float64, TFR_T_DECIMAL: np.float64, TFR_T_STRING: np.uint8,
               TFR_T_BINARY: np.uint8, TFR_T_NULL: np.uint8,
               TFR_T_BOOL: np.uint8, TFR_T_INT8: np.int8, TFR_T_INT16: np.int16, TFR_T_DATE: np.int32, TFR_T_TIMESTAMP: np.int64}


# RAGGED (include/tfrgpu.h): the schema flag of nestedArrayFormat=ragged and the two parts' feature-key suffixes
TFR_S_RAGGED = 0x1
TFR_RAGGED_VALUES_SUFFIX = "_values"
TFR_RAGGED_ROW_LENGTHS_SUFFIX = "_row_lengths"
# ... and of raggedPartition=rowSplits, with TFR_S_RAGGED: the partition stored as row splits
TFR_S_RAGGED_ROW_SPLITS = 0x8
TFR_RAGGED_ROW_SPLITS_SUFFIX = "_row_splits"
# INT64 TYPES (include/tfrgpu.h): the schema flag of extendedTypes=true
TFR_S_INT64_TYPES = 0x4


def make_fields(schema: StructType, vector_format: str = "dense", extended_types: bool = False):
    """StructType -> (ctypes array of tfr_field, keepalive list); VectorUDT fields by vector_format, BooleanType .. TimestampType
    by extended_types (lower_type)."""
    n = len(schema)
    arr = (tfr_field * max(n, 1))()
    keep = []
    for i, f in enumerate(schema):
        nm = f.name.encode("utf-8") if isinstance(f.name, str) else bytes(f.name)
        keep.append(nm)
        t, d = lower_type(f.dataType, vector_format, extended_types)
        arr[i].name = nm
        arr[i].name_len = len(nm)
        arr[i].elem_type = t
        arr[i].depth = d
        arr[i].nullable = 1 if f.nullable else 0
    return arr, keep


class HostColumn:
    """One column in the tfr_column layout, held as numpy arrays (host)."""

    __slots__ = ("elem_type", "depth", "n_levels", "n_rows", "null_count", "validity", "offsets", "values")

    def __init__(self, elem_type, depth, n_rows, validity, offsets, values, null_count=None):
        self.elem_type = elem_type
        self.depth = depth
        self.offsets = [np.ascontiguousarray(o, dtype=np.int32) for o in offsets]
        self.n_levels = len(self.offsets)
        self.n_rows = int(n_rows)
        self.validity = None if validity is None else np.ascontiguousarray(validity, dtype=np.uint8)
        self.values = np.ascontiguousarray(values, dtype=_LEAF_DTYPE[elem_type])
        if null_count is None:
            null_count = 0 if self.validity is None else int(self.n_rows - np.unpackbits(self.validity, bitorder="little")[: self.n_rows].sum())
        self.null_count = null_count

    def valid(self, r: int) -> bool:
        return self.validity is None or bool((self.validity[r >> 3] >> (r & 7)) & 1)

    # ---- row materialisation (what the JVM shim's row iterator does over the host copy) ----
    def _leaf(self, i):
        v = self.values[i]
        return v.item()

    def _leaf_range(self, lo, hi):
        if self.elem_type in (TFR_T_STRING, TFR_T_BINARY):
            so = self.offsets[-1]
            out = []
            for i in range(lo, hi):
                b = self.values[so[i]:so[i + 1]].tobytes()
                out.append(b.decode("utf-8") if self.elem_type == TFR_T_STRING else b)
            return out
        if self.elem_type in INT64_TYPES:
            return [int64_value(self.elem_type, v) for v in self.values[lo:hi].tolist()]
        return [v.item() for v in self.values[lo:hi]]

    def get(self, r: int):
        """Python value of row r: None, scalar, list or list of lists."""
        if self.elem_type == TFR_T_NULL or not self.valid(r):
            return None
        if self.depth == 0:
            return self._leaf_range(r, r + 1)[0]
        o0 = self.offsets[0]
        if self.depth == 1:
            return self._leaf_range(int(o0[r]), int(o0[r + 1]))
        o1 = self.offsets[1]
        return [self._leaf_range(int(o1[s]), int(o1[s + 1])) for s in range(int(o0[r]), int(o0[r + 1]))]

    def to_ctypes(self) -> tfr_column:
        c = tfr_column()
        c.elem_type = self.elem_type
        c.depth = self.depth
        c.n_levels = self.n_levels
        c.value_width = self.values.dtype.itemsize
        c.n_rows = self.n_rows
        c.null_count = self.null_count
        c.validity = None if self.validity is None else self.validity.ctypes.data
        for i, o in enumerate(self.offsets):
            c.offsets[i] = o.ctypes.data
            c.n_offsets[i] = len(o)
        c.values = self.values.ctypes.data
        c.n_values = len(self.values)
        return c

    def nbytes(self) -> int:
        n = 0 if self.validity is None else self.validity.nbytes
        return n + sum(o.nbytes for o in self.offsets) + self.values.nbytes


def column_from_ctypes(c: tfr_column) -> HostColumn:
    """Copy a host-pointer tfr_column into numpy-owned memory."""
    def arr(ptr, n, dt):
        if not ptr or n == 0:
            return np.zeros(0, dtype=dt)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(n * np.dtype(dt).itemsize,)).view(dt).copy()

    n_rows = c.n_rows
    validity = arr(c.validity, (n_rows + 7) // 8, np.uint8)
    offsets = [arr(c.offsets[i], c.n_offsets[i], np.int32) for i in range(c.n_levels)]
    values = arr(c.values, c.n_values, _LEAF_DTYPE[c.elem_type])
    return HostColumn(c.elem_type, c.depth, n_rows, validity, offsets, values, null_count=c.null_count)


def columns_from_rows(schema: StructType, rows: Sequence[Sequence], record_type: int = 0,
                      vector_format: str = "dense") -> List[HostColumn]:
    """Row-major Python values -> columnar HostColumns (what TFRecordOutputWriter buffers before
    handing a batch to tfr_encode).  Values follow Spark's external types: int, float, str,
    bytes, list, list of lists, a DenseVector or SparseVector for VectorUDT (its toArray, as a list<double> column; with
    vector_format="sparse", the columns of the lowered schema, filled from its toSparse); None = null."""
    sp = sparse_vector_fields(schema, vector_format)
    if sp:
        parts = [[sparse_parts(row[i]) for i in sp] for row in rows]
        lowered = [tuple(parts[r][sp.index(i)][1] if i in sp else v for i, v in enumerate(row)) +
                   tuple(x for p in parts[r] for x in (p[0], p[2])) for r, row in enumerate(rows)]
        return columns_from_rows(lowered_schema(schema, vector_format), lowered, record_type)
    cols = []
    n = len(rows)
    for ci, f in enumerate(schema):
        t, depth = lower_type(f.dataType, extended_types=True)   # (a schema without the option refused these types already)
        vector = t == TFR_T_VECTOR and depth == 0
        i64t = t in INT64_TYPES
        if vector:
            t, depth = TFR_T_FLOAT64, 1
        dt = _LEAF_DTYPE.get(t, np.uint8)
        varlen = t in (TFR_T_STRING, TFR_T_BINARY)
        nlev = depth + (1 if varlen else 0)
        offs = [[0] for _ in range(nlev)]
        leaves: list = []
        leafbytes = bytearray()
        valid = np.zeros((n + 7) // 8, dtype=np.uint8)

        def put_leaf(v):
            if varlen:
                b = v.encode("utf-8") if isinstance(v, str) else bytes(v)
                leafbytes.extend(b)
                offs[nlev - 1].append(len(leafbytes))
            else:
                leaves.append(int64_leaf(t, v) if i64t else v)

        def leaf_count():
            return (len(offs[nlev - 1]) - 1) if varlen else len(leaves)

        for r, row in enumerate(rows):
            v = row[ci]
            if v is None or t == TFR_T_NULL:
                if depth >= 1:
                    offs[0].append(offs[0][-1])
                elif varlen:
                    offs[0].append(offs[0][-1])
                else:
                    leaves.append(0)
                continue
            valid[r >> 3] |= 1 << (r & 7)
            if depth == 0:
                put_leaf(v)
            elif depth == 1:
                for e in (v.toArray().tolist() if vector else v):
                    put_leaf(e)
                offs[0].append(leaf_count())
            else:
                for inner in v:
                    for e in inner:
                        put_leaf(e)
                    offs[1].append(leaf_count())
                offs[0].append(len(offs[1]) - 1)
        if varlen:
            values = np.frombuffer(bytes(leafbytes), dtype=np.uint8)
        elif t in (TFR_T_INT32, TFR_T_INT64):
            # wrap to the column width like JVM int/long
            values = np.array([int(x) & ((1 << (8 * np.dtype(dt).itemsize)) - 1) for x in leaves], dtype=np.uint64).astype(
                np.uint32 if t == TFR_T_INT32 else np.uint64).view(dt)
        else:
            values = np.array(leaves, dtype=dt)
        cols.append(HostColumn(t, depth, n, valid, [np.array(o, dtype=np.int32) for o in offs], values))
    return cols
