"""ctypes binding of libtfrgpu.so (the C ABI in include/tfrgpu.h).

There is NO CPU fallback: if the shared library is missing, or no CUDA device is usable, creating a
decoder/encoder raises.  Nothing here imports or calls the oracle."""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional

import numpy as np

from . import _cabi as A
from ._cabi import HostColumn, column_from_ctypes, make_fields, tfr_batch_info, tfr_column, tfr_field
from .sqltypes import StructType

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TFR_LIB") or os.path.join(_DIR, "libtfrgpu.so")   # TFR_LIB: tuning builds only
_LIB = None

# every symbol include/tfrgpu.h declares
EXPORTS = [
    "tfr_abi_version", "tfr_status_string", "tfr_last_error", "tfr_schema_create", "tfr_schema_destroy",
    "tfr_schema_num_fields", "tfr_decoder_create", "tfr_decoder_create_permissive", "tfr_decoder_destroy", "tfr_decoder_staging", "tfr_decoder_staging_slot",
    "tfr_decoder_num_staging_slots", "tfr_decode", "tfr_decode_submit", "tfr_decode_at", "tfr_decode_submit_at", "tfr_batch_extent",
    "tfr_decoder_stream", "tfr_decoder_set_profiling", "tfr_decoder_get_profile", "tfr_decoder_get_stats", "tfr_batch_wait", "tfr_batch_status", "tfr_batch_consumed", "tfr_batch_dropped", "tfr_batch_dropped_spans", "tfr_batch_num_columns", "tfr_batch_columns",
    "tfr_batch_to_host_async", "tfr_batch_to_host", "tfr_batch_export_arrow_host", "tfr_batch_export_arrow_device", "tfr_batch_release",
    "tfr_batch_rows", "tfr_batch_rows_with_partition", "tfr_batch_rows_async",
    "tfr_encoder_create", "tfr_encoder_destroy", "tfr_encode", "tfr_encoder_row_staging", "tfr_encode_rows", "tfr_encoder_result_host",
    "tfr_encoder_stream", "tfr_encoder_num_row_slots", "tfr_encoder_row_staging_slot", "tfr_encode_rows_submit", "tfr_encoded_wait",
    "tfr_encoded_result", "tfr_encoded_release", "tfr_encoder_get_stats",
    "tfr_infer_create", "tfr_infer_create_mode", "tfr_infer_update", "tfr_infer_update_block", "tfr_infer_skipped",
    "tfr_infer_result", "tfr_infer_name", "tfr_infer_destroy",
]


class TfrError(RuntimeError):
    """Base of the exceptions mirroring what the reference throws (see INTEGRATION.md for the
    status -> Java exception table the JNI shim uses)."""
    java_class = "RuntimeException"

    def __init__(self, code: int, msg: str = "", row: int = -1, field: int = -1):
        self.code, self.row, self.field = code, row, field
        super().__init__(f"{self.java_class}: {msg or A.STATUS_NAMES.get(code, code)}"
                         + (f" (record {row})" if row >= 0 else "") + (f" (field {field})" if field >= 0 else ""))


class IOException(TfrError):
    java_class = "java.io.IOException"


class InvalidProtocolBufferException(IOException):
    java_class = "com.google.protobuf.InvalidProtocolBufferException"


class IllegalArgumentException(TfrError):
    java_class = "java.lang.IllegalArgumentException"


class NoSuchElementException(TfrError):
    java_class = "java.util.NoSuchElementException"


class NullPointerException(TfrError):
    java_class = "java.lang.NullPointerException"


class UnsupportedTypeException(TfrError):          # RuntimeException / UnsupportedOperationException
    java_class = "java.lang.RuntimeException"


class CudaError(TfrError):
    java_class = "java.lang.IllegalStateException"


_EXC = {
    A.TFR_E_CRC_LENGTH: IOException, A.TFR_E_CRC_DATA: IOException, A.TFR_E_TRUNCATED: IOException,
    A.TFR_E_RECORD_TOO_LARGE: IOException, A.TFR_E_MALFORMED_PROTO: InvalidProtocolBufferException,
    A.TFR_E_KIND_MISMATCH: IllegalArgumentException, A.TFR_E_BAD_RECORD_TYPE: IllegalArgumentException,
    A.TFR_E_EMPTY_SCALAR: NoSuchElementException, A.TFR_E_NULL_IN_NONNULL: NullPointerException,
    A.TFR_E_UNSUPPORTED_TYPE: UnsupportedTypeException, A.TFR_E_BAD_NESTING: UnsupportedTypeException,
    A.TFR_E_CUDA: CudaError,
}


def error_for(code: int, msg: str = "", row: int = -1, field: int = -1) -> TfrError:
    return _EXC.get(code, TfrError)(code, msg, row, field)


def lib():
    """Load libtfrgpu.so; raises (never falls back) when it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a).  There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i32, u32, i64, sz = C.c_void_p, C.c_int32, C.c_uint32, C.c_int64, C.c_size_t
    P = C.POINTER
    sig = {
        "tfr_abi_version": (i32, []),
        "tfr_status_string": (C.c_char_p, [i32]),
        "tfr_last_error": (C.c_char_p, []),
        "tfr_schema_create": (i32, [P(tfr_field), i32, i32, P(vp)]),
        "tfr_schema_destroy": (None, [vp]),
        "tfr_schema_num_fields": (i32, [vp]),
        "tfr_decoder_create": (i32, [vp, i32, u32, P(vp)]),
        "tfr_decoder_create_permissive": (i32, [vp, i32, u32, i32, P(vp)]),
        "tfr_decoder_destroy": (None, [vp]),
        "tfr_decoder_staging": (i32, [vp, sz, P(vp), P(sz)]),
        "tfr_decoder_staging_slot": (i32, [vp, i32, sz, P(vp), P(sz)]),
        "tfr_decoder_num_staging_slots": (i32, []),
        "tfr_decode": (i32, [vp, vp, sz, i32, i32, P(vp), P(sz)]),
        "tfr_decode_submit": (i32, [vp, vp, sz, i32, i32, P(vp)]),
        "tfr_decode_at": (i32, [vp, vp, sz, i32, i32, i64, i64, P(vp), P(sz)]),
        "tfr_decode_submit_at": (i32, [vp, vp, sz, i32, i32, i64, i64, P(vp)]),
        "tfr_batch_extent": (i32, [vp, P(C.c_size_t), P(i64)]),
        "tfr_decoder_get_stats": (i32, [vp, P(i64), i32]),
        "tfr_batch_to_host_async": (i32, [vp]),
        "tfr_infer_update_block": (i32, [vp, vp, sz, i32, i32, P(sz)]),
        "tfr_decoder_stream": (i32, [vp, P(vp)]),
        "tfr_decoder_set_profiling": (i32, [vp, i32]),
        "tfr_decoder_get_profile": (i32, [vp, P(C.c_double), P(i64), P(i64)]),
        "tfr_batch_wait": (i32, [vp]),
        "tfr_batch_status": (i32, [vp, P(tfr_batch_info)]),
        "tfr_batch_consumed": (i32, [vp, P(C.c_size_t)]),
        "tfr_batch_dropped": (i32, [vp, P(i64), P(i64), P(i64), P(i32), P(i32), i64]),
        "tfr_batch_dropped_spans": (i32, [vp, P(i64), P(i64), P(i64), P(i64), P(i32), P(i32), i64]),
        "tfr_batch_num_columns": (i32, [vp]),
        "tfr_batch_columns": (i32, [vp, P(tfr_column), i32]),
        "tfr_batch_to_host": (i32, [vp, P(tfr_column), i32]),
        "tfr_batch_export_arrow_host": (i32, [vp, i32, vp, vp]),
        "tfr_batch_export_arrow_device": (i32, [vp, i32, vp, vp]),
        "tfr_batch_release": (None, [vp]),
        "tfr_batch_rows": (i32, [vp, i32, P(vp), P(vp), P(i64), P(sz)]),
        "tfr_batch_rows_with_partition": (i32, [vp, i32, vp, sz, i32, vp, P(vp), P(vp), P(i64), P(sz)]),
        "tfr_batch_rows_async": (i32, [vp, i32, vp, sz, i32, vp]),
        "tfr_encoder_create": (i32, [vp, i32, u32, P(vp)]),
        "tfr_encoder_destroy": (None, [vp]),
        "tfr_encode": (i32, [vp, P(tfr_column), i32, i32, P(vp), P(sz), P(i64)]),
        "tfr_encoder_row_staging": (i32, [vp, sz, P(vp), P(sz)]),
        "tfr_encode_rows": (i32, [vp, vp, vp, i64, i32, P(vp), P(sz), P(i64)]),
        "tfr_encoder_result_host": (i32, [vp, P(vp), P(sz)]),
        "tfr_encoder_stream": (i32, [vp, P(vp)]),
        "tfr_encoder_num_row_slots": (i32, []),
        "tfr_encoder_row_staging_slot": (i32, [vp, i32, sz, P(vp), P(sz)]),
        "tfr_encode_rows_submit": (i32, [vp, vp, vp, i64, i32, P(vp)]),
        "tfr_encoded_wait": (i32, [vp, P(i64)]),
        "tfr_encoded_result": (i32, [vp, i32, P(vp), P(sz)]),
        "tfr_encoded_release": (None, [vp]),
        "tfr_encoder_get_stats": (i32, [vp, P(i64), i32]),
        "tfr_infer_create": (i32, [i32, i32, P(vp)]),
        "tfr_infer_create_mode": (i32, [i32, i32, u32, C.c_char_p, i32, P(vp)]),
        "tfr_infer_skipped": (i32, [vp, P(i64), P(i64), P(i64), P(i32), i64]),
        "tfr_infer_update": (i32, [vp, vp, sz, i32]),
        "tfr_infer_result": (i32, [vp, P(i32)]),
        "tfr_infer_name": (i32, [vp, i32, P(C.c_char_p), P(i32), P(i32)]),
        "tfr_infer_destroy": (None, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _LIB = L
    return L


def _check(rc: int):
    if rc != 0:
        msg = lib().tfr_last_error()
        raise error_for(rc, msg.decode("utf-8", "replace") if msg else "")


class Schema:
    def __init__(self, schema: StructType, record_type: int = 0, vector_format: str = "dense"):
        """`vector_format`: the `vectorFormat` option, how VectorUDT fields are stored (include/tfrgpu.h, VECTORS and SPARSE
        VECTORS); "sparse" lowers each to three fields (sqltypes.lowered_schema), and the columns follow the lowered schema"""
        self.struct = schema
        self.record_type = record_type
        self.vector_format = vector_format
        fields, self._keep = make_fields(schema, vector_format)
        h = C.c_void_p()
        _check(lib().tfr_schema_create(fields, len(schema), record_type, C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            lib().tfr_schema_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _device_ptr(obj):
    """(ptr, nbytes, on_device, keepalive) for bytes / numpy / torch tensors"""
    try:
        import torch
        if isinstance(obj, torch.Tensor):
            t = obj.contiguous()
            return t.data_ptr(), t.numel() * t.element_size(), 1 if t.is_cuda else 0, t
    except ImportError:
        pass
    if isinstance(obj, np.ndarray):
        a = np.ascontiguousarray(obj)
        return a.ctypes.data, a.nbytes, 0, a
    if isinstance(obj, (bytes, bytearray, memoryview)):
        a = np.frombuffer(obj, dtype=np.uint8)
        return a.ctypes.data, a.nbytes, 0, a
    if isinstance(obj, tuple) and len(obj) == 3:     # (ptr, nbytes, on_device)
        return obj[0], obj[1], obj[2], None
    raise TypeError(type(obj))


class Batch:
    """A decoded batch.  After Decoder.submit() the result is not known yet: `info` / `n_rows` (and every accessor
    below) wait for it on first use (tfr_batch_status resolves a pipelined batch)."""

    def __init__(self, h, ncols, keep=None):
        self.h = h
        self.ncols = ncols
        self._info = None
        self._keep = keep          # the input buffer of a pipelined batch must outlive it

    @property
    def info(self) -> dict:
        if self._info is None:
            info = tfr_batch_info()
            _check(lib().tfr_batch_status(self.h, C.byref(info)))
            self._info = {k: getattr(info, k) for k, _ in tfr_batch_info._fields_}
        return self._info

    @property
    def n_rows(self) -> int:
        return self.info["n_rows"]

    def wait(self):
        _check(lib().tfr_batch_wait(self.h))

    def consumed(self) -> int:
        """bytes of the submitted block this batch consumes: known once the frame index has run, before the rows are decoded"""
        n = C.c_size_t()
        _check(lib().tfr_batch_consumed(self.h, C.byref(n)))
        return n.value

    def extent(self) -> tuple:
        """(consumed bytes, entries in them) with consumed()'s wait (tfr_batch_extent): a streaming reader adds them to the
        next block's first_offset and first_entry"""
        n, e = C.c_size_t(), C.c_int64()
        _check(lib().tfr_batch_extent(self.h, C.byref(n), C.byref(e)))
        return n.value, e.value

    def dropped(self) -> List[tuple]:
        """the records a drop-mode decoder (TFR_F_DROP_MALFORMED) cut out of this batch, or a PERMISSIVE one delivered as
        corrupt rows, in record order (tfr_batch_dropped):
        [(frame index in the block, byte offset in the submitted buffer, TFR_E_* code, schema field or -1)]"""
        return [(rec, off, code, field) for rec, off, _, code, field in self.dropped_spans()]

    def dropped_spans(self) -> List[tuple]:
        """dropped() with each entry's byte length (tfr_batch_dropped_spans): 16 + L for a frame, p - o for a lost region
        (TFR_F_RESYNC): [(entry index in the block, byte offset in the submitted buffer, byte length, TFR_E_* code, field)]"""
        n = C.c_int64()
        _check(lib().tfr_batch_dropped_spans(self.h, C.byref(n), None, None, None, None, None, 0))
        k = n.value
        if k == 0:
            return []
        rec, off, nb = (C.c_int64 * k)(), (C.c_int64 * k)(), (C.c_int64 * k)()
        code, field = (C.c_int32 * k)(), (C.c_int32 * k)()
        _check(lib().tfr_batch_dropped_spans(self.h, C.byref(n), rec, off, nb, code, field, k))
        return [(rec[i], off[i], nb[i], code[i], field[i]) for i in range(k)]

    def to_host_async(self):
        """enqueue the D2H of every Arrow buffer behind the batch's kernels (overlaps the next batch)"""
        _check(lib().tfr_batch_to_host_async(self.h))

    def device_columns(self) -> List[tfr_column]:
        cols = (tfr_column * max(self.ncols, 1))()
        _check(lib().tfr_batch_columns(self.h, cols, self.ncols))
        return [cols[i] for i in range(self.ncols)]

    def to_host_raw(self):
        """D2H into the batch's pinned buffer; returns ctypes columns with host pointers (zero extra copy)"""
        cols = (tfr_column * max(self.ncols, 1))()
        _check(lib().tfr_batch_to_host(self.h, cols, self.ncols))
        return [cols[i] for i in range(self.ncols)]

    def to_host(self) -> List[HostColumn]:
        return [column_from_ctypes(c) for c in self.to_host_raw()]

    def to_arrow(self):
        """pyarrow arrays through the Arrow C Data Interface export"""
        import pyarrow as pa
        from pyarrow.cffi import ffi
        out = []
        for i in range(self.ncols):
            ca = ffi.new("struct ArrowArray*")
            cs = ffi.new("struct ArrowSchema*")
            _check(lib().tfr_batch_export_arrow_host(self.h, i, int(ffi.cast("uintptr_t", ca)), int(ffi.cast("uintptr_t", cs))))
            out.append(pa.Array._import_from_c(int(ffi.cast("uintptr_t", ca)), int(ffi.cast("uintptr_t", cs))))
        return out

    def unsafe_rows(self, to_host: bool = True, partition=None):
        """The batch's rows as Spark UnsafeRows (tfr_batch_rows).  to_host=True: (uint8 rows, int64 offsets[n_rows + 1]),
        numpy views of pinned memory the batch owns (valid until release).  to_host=False: (rows device ptr, offsets device
        ptr, n_rows, nbytes).  Raises UnsupportedTypeException for a schema with a DecimalType field.
        partition=(row_bytes, var_flags) appends a file's partition values to every row (tfr_batch_rows_with_partition):
        row_bytes is the UnsafeRow of the partition schema alone, var_flags one 0 / 1 per partition field (1: String,
        Binary, Decimal with precision > 18)."""
        rp, op = C.c_void_p(), C.c_void_p()
        n, nb = C.c_int64(), C.c_size_t()
        if partition is None:
            _check(lib().tfr_batch_rows(self.h, 1 if to_host else 0, C.byref(rp), C.byref(op), C.byref(n), C.byref(nb)))
        else:
            row, flags = bytes(partition[0]), bytes(bytearray(partition[1]))
            _check(lib().tfr_batch_rows_with_partition(self.h, 1 if to_host else 0, row, len(row), len(flags), flags,
                                                       C.byref(rp), C.byref(op), C.byref(n), C.byref(nb)))
        if not to_host:
            return rp.value or 0, op.value or 0, n.value, nb.value
        rows = np.ctypeslib.as_array(C.cast(rp, C.POINTER(C.c_uint8)), shape=(nb.value,)) if nb.value else np.zeros(0, np.uint8)
        offs = np.ctypeslib.as_array(C.cast(op, C.POINTER(C.c_int64)), shape=(n.value + 1,))
        return rows, offs

    def unsafe_rows_async(self, to_host: bool = True, partition=None):
        """Enqueue the rows unsafe_rows() returns, and with to_host their copy to pinned memory, behind the batch's kernels
        without waiting (tfr_batch_rows_async); unsafe_rows() then reads them.  partition as in unsafe_rows()."""
        if partition is None:
            _check(lib().tfr_batch_rows_async(self.h, 1 if to_host else 0, None, 0, 0, None))
        else:
            row, flags = bytes(partition[0]), bytes(bytearray(partition[1]))
            _check(lib().tfr_batch_rows_async(self.h, 1 if to_host else 0, row, len(row), len(flags), flags))

    def raise_if_error(self):
        if self.info["error_code"]:
            raise error_for(self.info["error_code"], "", self.info["error_row"], self.info["error_field"])

    def release(self):
        if self.h:
            lib().tfr_batch_release(self.h)
            self.h = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class Decoder:
    def __init__(self, schema: StructType, record_type: int = 0, device: int = 0, flags: int = A.TFR_F_DEFAULT,
                 corrupt_field: Optional[int] = None, vector_format: str = "dense"):
        """`corrupt_field`: with TFR_F_PERMISSIVE in `flags`, the index of the schema field that receives a failing record's
        payload (a nullable BinaryType column; tfr_decoder_create_permissive).  `vector_format`: as Schema's."""
        self.schema = Schema(schema, record_type, vector_format)
        self.ncols = lib().tfr_schema_num_fields(self.schema.h)     # ByteArray: byteArray, then the generated fields
        h = C.c_void_p()
        if corrupt_field is None:
            _check(lib().tfr_decoder_create(self.schema.h, device, flags, C.byref(h)))
        else:
            _check(lib().tfr_decoder_create_permissive(self.schema.h, device, flags, corrupt_field, C.byref(h)))
        self.h = h

    def staging(self, nbytes: int) -> np.ndarray:
        p = C.c_void_p()
        cap = C.c_size_t()
        _check(lib().tfr_decoder_staging(self.h, nbytes, C.byref(p), C.byref(cap)))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(cap.value,))

    def staging_slot(self, slot: int, nbytes: int) -> np.ndarray:
        p = C.c_void_p()
        cap = C.c_size_t()
        _check(lib().tfr_decoder_staging_slot(self.h, slot, nbytes, C.byref(p), C.byref(cap)))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(cap.value,))

    @staticmethod
    def num_staging_slots() -> int:
        return lib().tfr_decoder_num_staging_slots()

    def stats(self) -> dict:
        v = (C.c_int64 * 14)()
        _check(lib().tfr_decoder_get_stats(self.h, v, 14))
        names = ["batches", "speculative_submits", "speculative_redone", "count_mode_batches", "general_path_batches", "shapes_learned", "transcode_reruns",
                 "rows_async", "rows_async_rebuilt", "records_dropped", "records_corrupt"]
        names += ["lost_regions", "lost_region_bytes"]                   # TFR_F_RESYNC
        names += ["large_record_batches"]                               # the large-record kernel (csrc/large.cuh)
        return {k: v[i] for i, k in enumerate(names)}

    def stream(self) -> int:
        p = C.c_void_p()
        _check(lib().tfr_decoder_stream(self.h, C.byref(p)))
        return p.value or 0

    def set_profiling(self, enable: bool):
        _check(lib().tfr_decoder_set_profiling(self.h, 1 if enable else 0))

    def get_profile(self):
        ms = (C.c_double * 8)()
        nl = C.c_int64()
        n1 = C.c_int64()
        _check(lib().tfr_decoder_get_profile(self.h, ms, C.byref(nl), C.byref(n1)))
        names = ["frame_index", "pass1", "scan", "pass2", "pack_validity", "h2d", "d2h", "rows"]
        return {"ms": {k: ms[i] for i, k in enumerate(names)}, "launches": nl.value, "pass1_launches": n1.value}

    def decode(self, data, is_final: bool = True, nbytes: Optional[int] = None, first_entry: int = 0, first_offset: int = 0):
        """-> (Batch, consumed_bytes).  first_entry / first_offset: the block's position in its file, the base of the
        generated fields (tfr_decode_at)"""
        ptr, n, on_dev, keep = _device_ptr(data)
        if nbytes is not None:
            n = nbytes
        b = C.c_void_p()
        used = C.c_size_t()
        _check(lib().tfr_decode_at(self.h, ptr, n, on_dev, 1 if is_final else 0, first_entry, first_offset, C.byref(b), C.byref(used)))
        return Batch(b, self.ncols), used.value

    def submit(self, data, is_final: bool = True, nbytes: Optional[int] = None, first_entry: int = 0,
               first_offset: int = 0) -> "Batch":
        """pipelined decode (tfr_decode_submit_at): returns at once; Batch.info["consumed_bytes"] has the consumed count"""
        ptr, n, on_dev, keep = _device_ptr(data)
        if nbytes is not None:
            n = nbytes
        b = C.c_void_p()
        _check(lib().tfr_decode_submit_at(self.h, ptr, n, on_dev, 1 if is_final else 0, first_entry, first_offset, C.byref(b)))
        return Batch(b, self.ncols, keep)

    def close(self):
        if self.h:
            lib().tfr_decoder_destroy(self.h)
            self.h = None
        self.schema.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Encoder:
    def __init__(self, schema: StructType, record_type: int = 0, device: int = 0, flags: int = 0, vector_format: str = "dense"):
        self.schema = Schema(schema, record_type, vector_format)
        self.ncols = 1 if record_type == 2 else lib().tfr_schema_num_fields(self.schema.h)   # (a sparse vector adds two)
        h = C.c_void_p()
        _check(lib().tfr_encoder_create(self.schema.h, device, flags, C.byref(h)))
        self.h = h

    def encode_columns(self, cols: List[tfr_column], on_device: bool):
        """-> (device ptr, nbytes); raises NullPointerException for a null in a non-nullable column"""
        arr = (tfr_column * max(len(cols), 1))(*cols)
        out = C.c_void_p()
        nb = C.c_size_t()
        er = C.c_int64(-1)
        rc = lib().tfr_encode(self.h, arr, len(cols), 1 if on_device else 0, C.byref(out), C.byref(nb), C.byref(er))
        if rc != 0:
            msg = lib().tfr_last_error()
            raise error_for(rc, msg.decode("utf-8", "replace") if msg else "", er.value)
        return out.value or 0, nb.value

    def encode(self, columns: List[HostColumn]) -> bytes:
        cols = [c.to_ctypes() for c in columns]
        self.encode_columns(cols, False)
        return self.result_host()

    def row_staging(self, nbytes: int) -> np.ndarray:
        """pinned host memory for UnsafeRow bytes (tfr_encoder_row_staging); valid until a call that needs more"""
        p = C.c_void_p()
        cap = C.c_size_t()
        _check(lib().tfr_encoder_row_staging(self.h, nbytes, C.byref(p), C.byref(cap)))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(cap.value,))

    def encode_rows(self, rows, offsets, on_device: Optional[bool] = None):
        """Spark UnsafeRows -> (device ptr, nbytes) of the framed records (tfr_encode_rows).  rows: the row bytes, offsets:
        n_rows + 1 int32 row starts; numpy / bytes (host) or torch tensors (host or CUDA).  Raises TfrError with code
        TFR_E_INVALID_ARG for a malformed row and NullPointerException for a null the writer cannot take; .row is the row."""
        rp, _, rdev, keep_r = _device_ptr(rows)
        if not isinstance(offsets, tuple):
            try:
                import torch
                is_t = isinstance(offsets, torch.Tensor)
            except ImportError:
                is_t = False
            offsets = offsets.to(torch.int32) if is_t else np.asarray(offsets, dtype=np.int32)
        op, onb, odev, keep_o = _device_ptr(offsets)
        if rdev != odev:
            raise ValueError("rows and offsets must both be host or both be device memory")
        n_rows = onb // 4 - 1 if not isinstance(offsets, tuple) else offsets[1] // 4 - 1
        dev = rdev if on_device is None else (1 if on_device else 0)
        out = C.c_void_p()
        nb = C.c_size_t()
        er = C.c_int64(-1)
        rc = lib().tfr_encode_rows(self.h, rp, op, max(n_rows, 0), dev, C.byref(out), C.byref(nb), C.byref(er))
        if rc != 0:
            msg = lib().tfr_last_error()
            raise error_for(rc, msg.decode("utf-8", "replace") if msg else "", er.value)
        return out.value or 0, nb.value

    def result_host(self) -> bytes:
        p = C.c_void_p()
        nb = C.c_size_t()
        _check(lib().tfr_encoder_result_host(self.h, C.byref(p), C.byref(nb)))
        return C.string_at(p, nb.value)

    @staticmethod
    def num_row_slots() -> int:
        return lib().tfr_encoder_num_row_slots()

    def row_staging_slot(self, slot: int, nbytes: int) -> np.ndarray:
        """pinned row staging of pipeline slot `slot` (slot 0 is row_staging); refill it once the submission that read it
        has been waited on or released"""
        p = C.c_void_p()
        cap = C.c_size_t()
        _check(lib().tfr_encoder_row_staging_slot(self.h, slot, nbytes, C.byref(p), C.byref(cap)))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(cap.value,))

    def submit_rows(self, rows, offsets, on_device: Optional[bool] = None) -> "Encoded":
        """pipelined encode_rows (tfr_encode_rows_submit): returns at once; Encoded.wait() raises what encode_rows raises"""
        rp, _, rdev, keep_r = _device_ptr(rows)
        if not isinstance(offsets, tuple):
            try:
                import torch
                is_t = isinstance(offsets, torch.Tensor)
            except ImportError:
                is_t = False
            offsets = offsets.to(torch.int32) if is_t else np.asarray(offsets, dtype=np.int32)
        op, onb, odev, keep_o = _device_ptr(offsets)
        if rdev != odev:
            raise ValueError("rows and offsets must both be host or both be device memory")
        n_rows = onb // 4 - 1 if not isinstance(offsets, tuple) else offsets[1] // 4 - 1
        dev = rdev if on_device is None else (1 if on_device else 0)
        h = C.c_void_p()
        _check(lib().tfr_encode_rows_submit(self.h, rp, op, max(n_rows, 0), dev, C.byref(h)))
        return Encoded(h, self, (keep_r, keep_o))

    def stats(self) -> dict:
        v = (C.c_int64 * 8)()
        _check(lib().tfr_encoder_get_stats(self.h, v, 8))
        names = ["submits", "speculative_submits", "speculative_redone", "host_topups", "general_emit"]
        return {k: v[i] for i, k in enumerate(names)}

    def stream(self) -> int:
        p = C.c_void_p()
        _check(lib().tfr_encoder_stream(self.h, C.byref(p)))
        return p.value or 0

    def close(self):
        if self.h:
            lib().tfr_encoder_destroy(self.h)
            self.h = None
        self.schema.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Encoded:
    """One pipelined encode (Encoder.submit_rows).  Every accessor waits for it first; the bytes stay valid until release()."""

    def __init__(self, h, enc, keep=None):
        self.h = h
        self.enc = enc
        self._keep = keep          # the input of a pending submission must outlive it

    def wait(self):
        """raises the TfrError subclass (with .row) encode_rows raises for the same rows"""
        er = C.c_int64(-1)
        rc = lib().tfr_encoded_wait(self.h, C.byref(er))
        if rc != 0:
            msg = lib().tfr_last_error()
            raise error_for(rc, msg.decode("utf-8", "replace") if msg else "", er.value)

    def _result(self, to_host: int):
        self.wait()
        p = C.c_void_p()
        nb = C.c_size_t()
        _check(lib().tfr_encoded_result(self.h, to_host, C.byref(p), C.byref(nb)))
        return p.value or 0, nb.value

    def result_host(self) -> bytes:
        p, n = self._result(1)
        return C.string_at(p, n) if n else b""

    def result_device(self):
        """-> (device ptr, nbytes)"""
        return self._result(0)

    def release(self):
        # after Encoder.close() the encoder has freed every submission already
        if self.h and self.enc.h:
            lib().tfr_encoded_release(self.h)
        self.h = None
        self._keep = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class Infer:
    """Schema inference accumulator (tfr_infer_*): update() is the seqOp over one block of framed bytes, result()
    the merged name -> lattice code map (TFR_INF_*).  `flags` picks the parse mode (0: FAILFAST; TFR_F_DROP_MALFORMED or
    TFR_F_PERMISSIVE skip failing records, see skipped()); PERMISSIVE takes the corrupt-record column's name, which
    inference ignores in every record (tfr_infer_create_mode)."""

    def __init__(self, record_type: int = 0, device: int = 0, flags: int = 0, corrupt_name=None):
        h = C.c_void_p()
        self.h = None
        name = corrupt_name.encode() if isinstance(corrupt_name, str) else corrupt_name
        _check(lib().tfr_infer_create_mode(record_type, device, flags, name, len(name) if name is not None else 0, C.byref(h)))
        self.h = h

    def update(self, data):
        ptr, n, on_dev, keep = _device_ptr(data)
        _check(lib().tfr_infer_update(self.h, ptr, n, on_dev))

    def update_block(self, data, is_final: bool, nbytes: Optional[int] = None) -> int:
        """one block of a streamed file (tfr_infer_update_block) -> consumed bytes"""
        ptr, n, on_dev, keep = _device_ptr(data)
        if nbytes is not None:
            n = nbytes
        used = C.c_size_t()
        _check(lib().tfr_infer_update_block(self.h, ptr, n, on_dev, 1 if is_final else 0, C.byref(used)))
        return used.value

    def skipped(self) -> List[tuple]:
        """the records the last update call skipped, in record order (tfr_infer_skipped), shaped like Batch.dropped():
        [(frame index in the block, byte offset in the submitted buffer, TFR_E_* code, -1)]"""
        n = C.c_int64()
        _check(lib().tfr_infer_skipped(self.h, C.byref(n), None, None, None, 0))
        k = n.value
        if k == 0:
            return []
        rec, off, code = (C.c_int64 * k)(), (C.c_int64 * k)(), (C.c_int32 * k)()
        _check(lib().tfr_infer_skipped(self.h, C.byref(n), rec, off, code, k))
        return [(rec[i], off[i], code[i], -1) for i in range(k)]

    def result(self) -> dict:
        n = C.c_int32()
        _check(lib().tfr_infer_result(self.h, C.byref(n)))
        out = {}
        for i in range(n.value):
            nm = C.c_char_p(); ln = C.c_int32(); code = C.c_int32()
            _check(lib().tfr_infer_name(self.h, i, C.byref(nm), C.byref(ln), C.byref(code)))
            out[C.string_at(nm, ln.value)] = code.value
        return out

    def close(self):
        if self.h:
            lib().tfr_infer_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
