"""Host-side mirror of the reference interface for the hot path, by name.

    reference (Scala)                                   here
    ------------------------------------------------    ---------------------------------------------
    TFRecordFileReader.readFile(conf, options, file,    TFRecordFileReader.readFile(conf, options, file, schema)
        schema): Iterator[InternalRow]                      -> iterator of row tuples
        (M/TFRecordFileReader.scala:16-83)
    new TFRecordDeserializer(schema).deserializeExample TFRecordDeserializer(schema).deserializeExample(bytes)
        (M/TFRecordDeserializer.scala:21-61)
    new TFRecordSerializer(schema).serializeExample     TFRecordSerializer(schema).serializeExample(row) -> bytes
        (M/TFRecordSerializer.scala:20-60)
    new TFRecordOutputWriter(path, options, schema,     TFRecordOutputWriter(path, options, dataSchema, context)
        context).write(row)/close()                         .write(row) / .close()
        (M/TFRecordOutputWriter.scala:12-44)
    DefaultSource (M/DefaultSource.scala:23-143)        DefaultSource: shortName/isSplitable/buildReader/prepareWrite

Everything that touches record bytes goes through the C ABI (libtfrgpu.so): there is no Python or CPU
implementation of the path in this package.  Rows are tuples of Python values (None, int, float, str,
bytes, list, list of lists) standing in for Catalyst's InternalRow; message arguments are serialized
protobuf bytes (there are no org.tensorflow.example classes here)."""
from __future__ import annotations

import logging
import os
import struct
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np

from . import _cabi, _native
from ._cabi import TFR_F_DEFAULT, TFR_F_DROP_MALFORMED, TFR_F_PERMISSIVE, TFR_F_RESYNC, TFR_E_BATCH_TOO_LARGE as A_TFR_E_BATCH_TOO_LARGE, columns_from_rows
from .sqltypes import (RECORD_TYPES, BinaryType, DenseVector, LongType, RecordOffsetType, RowIndexType, SparseVector, StructField,
                       StructType, VectorUDT, byte_array_schema, check_vector_format, sparse_vector_fields)

M = "src/main/scala/com/linkedin/spark/datasources/tfrecord/"
_LOG = logging.getLogger(__name__)


# Spark's generated metadata fields (FileFormat.ROW_INDEX, ROW_INDEX_TEMPORARY_COLUMN_NAME in Spark 3.4 / 3.5; restated, not
# checked against a JVM): `_metadata.row_index` is filled by the reader through a temporary LongType column that Spark adds
# to the required schema.  record_offset follows the same pattern.  The decoder fills both on the GPU (include/tfrgpu.h,
# POSITIONS).
ROW_INDEX, ROW_INDEX_TEMPORARY_COLUMN_NAME = "row_index", "_tmp_metadata_row_index"
RECORD_OFFSET, RECORD_OFFSET_TEMPORARY_COLUMN_NAME = "record_offset", "_tmp_metadata_record_offset"
_GENERATED = {ROW_INDEX_TEMPORARY_COLUMN_NAME: RowIndexType(), RECORD_OFFSET_TEMPORARY_COLUMN_NAME: RecordOffsetType()}


def _decoder_schema(requiredSchema: StructType) -> StructType:
    """the required schema as the decoder takes it: Spark's temporary metadata columns (LongType) become generated fields,
    at their place; every other field is a data field"""
    return StructType([StructField(f.name, _GENERATED[f.name], False) if f.name in _GENERATED and f.dataType == LongType() else f
                       for f in requiredSchema])


def _record_type(options: Optional[Dict[str, str]]) -> int:
    rt = (options or {}).get("recordType", "Example")          # M/TFRecordFileReader.scala:22
    if rt not in RECORD_TYPES:                                  # :78-79
        raise _native.IllegalArgumentException(-3, f"Unsupported recordType {rt}: recordType can be ByteArray, Example or SequenceExample")
    return RECORD_TYPES[rt]


def _vector_format(options: Optional[Dict[str, str]]) -> str:
    """the `vectorFormat` option: how VectorUDT fields are stored.  "dense" (the default): the FloatList of toArray under the
    field's name; "sparse": the TF sparse features <name>_indices, <name>_values and <name>_size of toSparse (include/tfrgpu.h,
    SPARSE VECTORS).  Anything else is refused before any work."""
    vf = (options or {}).get("vectorFormat", "dense")
    try:
        return check_vector_format(vf)
    except ValueError as e:
        raise _native.IllegalArgumentException(-1, str(e)) from None


def _corrupt_column_name(options: Optional[Dict[str, str]]) -> str:
    """the option columnNameOfCorruptRecord, named and defaulted as Spark's JSON and CSV sources have it"""
    return (options or {}).get("columnNameOfCorruptRecord", "_corrupt_record")


def _parse_mode(options: Optional[Dict[str, str]]) -> str:
    """the `mode` option, case-insensitive as Spark's ParseMode reads it -> FAILFAST, DROPMALFORMED or PERMISSIVE"""
    mode = (options or {}).get("mode", "FAILFAST")
    m = mode.upper() if isinstance(mode, str) else mode
    if m in ("FAILFAST", "DROPMALFORMED", "PERMISSIVE"):
        return m
    raise _native.IllegalArgumentException(-1, f"mode {mode}: the tfrecord source supports FAILFAST and DROPMALFORMED, and "
                                               f"PERMISSIVE with a corrupt-record column")


def _resync_flag(options: Optional[Dict[str, str]], mode: str) -> int:
    """the `resyncFraming` option ("false" by default, or "true", case-insensitive) -> 0 or TFR_F_RESYNC: after a framing
    error (a bad length CRC, a length above 2^31 - 1, a record cut off at the end of the file) reading goes on at the next
    record whose two CRCs verify, instead of failing the file.  DROPMALFORMED drops the bytes in between, PERMISSIVE reads
    them as one corrupt row.  Only with those two modes: FAILFAST is the reference's behaviour and stays so."""
    value = (options or {}).get("resyncFraming", "false")
    v = value.lower() if isinstance(value, str) else value
    if v not in ("true", "false"):
        raise _native.IllegalArgumentException(-1, f"resyncFraming {value}: the option takes true or false")
    if v == "false":
        return 0
    if mode not in ("DROPMALFORMED", "PERMISSIVE"):
        raise _native.IllegalArgumentException(-1, f"resyncFraming needs mode DROPMALFORMED or PERMISSIVE (mode {mode})")
    return TFR_F_RESYNC


_MODE_FLAGS = {"FAILFAST": TFR_F_DEFAULT, "DROPMALFORMED": TFR_F_DEFAULT | TFR_F_DROP_MALFORMED, "PERMISSIVE": TFR_F_DEFAULT | TFR_F_PERMISSIVE}


def _mode_flags(options: Optional[Dict[str, str]]) -> Tuple[str, int]:
    """the `mode` and `resyncFraming` options -> (mode, flags of the decoder and of schema inference)"""
    m = _parse_mode(options)
    return m, _MODE_FLAGS[m] | _resync_flag(options, m)


def _decoder_flags(options: Optional[Dict[str, str]], dataSchema: Optional[StructType] = None) -> int:
    """the `mode` option -> decoder flags.  FAILFAST (the default, the reference's behaviour): the first failing record
    ends the file.  DROPMALFORMED: failing records are dropped and the rest is read (framing errors still end the file).
    PERMISSIVE: a failing record is read as a row of nulls; it needs a corrupt-record column in `dataSchema` (a field
    named by columnNameOfCorruptRecord, nullable BinaryType), which receives the record's payload, and Example or
    SequenceExample records.  resyncFraming=true (DROPMALFORMED and PERMISSIVE only) adds TFR_F_RESYNC."""
    m, flags = _mode_flags(options)
    if m == "PERMISSIVE":
        name = _corrupt_column_name(options)
        field = next((f for f in dataSchema or () if f.name == name), None)
        if field is None:
            raise _native.IllegalArgumentException(-1, f"mode PERMISSIVE needs a corrupt-record column: the data schema has no field "
                                                       f"'{name}' (option columnNameOfCorruptRecord); use FAILFAST or DROPMALFORMED")
        if field.dataType != BinaryType() or not field.nullable:
            raise _native.IllegalArgumentException(-1, f"The field for corrupt records must be binary type and nullable: '{name}' "
                                                       f"is {field.dataType!r}{'' if field.nullable else ' NOT NULL'}")
        if _record_type(options) == RECORD_TYPES["ByteArray"]:
            raise _native.IllegalArgumentException(-1, "mode PERMISSIVE: ByteArray records have no corrupt-record column; "
                                                       "use FAILFAST or DROPMALFORMED")
    return flags


def _read_mode(options: Optional[Dict[str, str]], dataSchema: StructType, requiredSchema: StructType):
    """-> (decoder flags, index of the corrupt-record column in `requiredSchema` or None).  PERMISSIVE with that column
    pruned by a projection still reads failing records, as rows of nulls (Spark's JSON source does the same)."""
    flags = _decoder_flags(options, dataSchema)
    if not flags & TFR_F_PERMISSIVE:
        return flags, None
    name = _corrupt_column_name(options)
    return flags, next((i for i, f in enumerate(requiredSchema) if f.name == name), None)


# ---- stream compression (SURVEY 8f.3): host-side, around the same GPU kernels -------------------------------------------
# The reference hands `codec` to Hadoop (M/DefaultSource.scala:94-102: a codec class name) and CodecStreams compresses the
# whole output stream; on read, Hadoop picks the codec from the file extension.  The compressed bytes are a container
# around the framed records, so they are (de)compressed on the host and the framed bytes go through the C ABI unchanged.
_CODECS = {   # name -> (file extension, Hadoop class)
    "gzip": (".gz", "org.apache.hadoop.io.compress.GzipCodec"),
    "deflate": (".deflate", "org.apache.hadoop.io.compress.DefaultCodec"),
    "bzip2": (".bz2", "org.apache.hadoop.io.compress.BZip2Codec"),
}


def _codec_name(codec: str) -> Optional[str]:
    """option value (Hadoop class name, or its short name) -> one of _CODECS; '' -> None"""
    if not codec:
        return None
    for name, (_, cls) in _CODECS.items():
        if codec == cls or codec.lower() == name or codec.lower() == cls.rsplit(".", 1)[1].lower():
            return name
    raise _native.IllegalArgumentException(-3, f"codec {codec}: only GzipCodec, DefaultCodec (deflate) and BZip2Codec are available on this host")


def _codec_of_path(path: str) -> Optional[str]:
    for name, (ext, _) in _CODECS.items():
        if path.endswith(ext):
            return name
    return None


class _DeflateReader:
    """zlib-format stream (Hadoop DefaultCodec, '.deflate') as a file-like object with read(n)"""

    def __init__(self, f):
        import zlib
        self._f, self._z, self._buf, self._eof = f, zlib.decompressobj(), b"", False

    def read(self, n: int = -1) -> bytes:
        while not self._eof and (n < 0 or len(self._buf) < n):
            raw = self._f.read(1 << 20)
            if not raw:
                self._buf += self._z.flush()
                self._eof = True
                break
            self._buf += self._z.decompress(raw)
        if n < 0:
            out, self._buf = self._buf, b""
        else:
            out, self._buf = self._buf[:n], self._buf[n:]
        return out

    def close(self):
        self._f.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class _DeflateWriter:
    def __init__(self, f):
        import zlib
        self._f, self._z = f, zlib.compressobj()

    def write(self, b: bytes):
        self._f.write(self._z.compress(b))

    def close(self):
        self._f.write(self._z.flush())
        self._f.close()


def _open_read(path: str):
    """file object yielding the FRAMED bytes of `path` (decompressed when the extension names a codec)"""
    codec = _codec_of_path(path)
    if codec == "gzip":
        import gzip
        return gzip.open(path, "rb")
    if codec == "bzip2":
        import bz2
        return bz2.open(path, "rb")
    if codec == "deflate":
        return _DeflateReader(open(path, "rb"))
    return open(path, "rb")


def _open_write(path: str, codec: Optional[str]):
    if codec == "gzip":
        import gzip
        return gzip.open(path, "wb")
    if codec == "bzip2":
        import bz2
        return bz2.open(path, "wb")
    if codec == "deflate":
        return _DeflateWriter(open(path, "wb"))
    return open(path, "wb")


def _rows_of(batch: "_native.Batch", schema: Optional[StructType] = None, vector_format: str = "dense") -> List[tuple]:
    """the batch's rows; a VectorUDT field of `schema` (the decoder's, Example or SequenceExample) becomes a DenseVector, or
    with vector_format="sparse" a SparseVector of its three lowered columns (null when its values are), whose constructor
    checks what the decoder does not (SPARSE VECTORS)"""
    cols = batch.to_host()
    if schema is None:
        return [tuple(c.get(r) for c in cols) for r in range(batch.n_rows)]
    nf = len(schema)
    sp = {i: nf + 2 * j for j, i in enumerate(sparse_vector_fields(schema, vector_format))}
    vec = [isinstance(f.dataType, VectorUDT) for f in schema]

    def value(i, r):
        v = cols[i].get(r)
        if v is None or not vec[i]:
            return v
        if i not in sp:
            return DenseVector(v)
        idx, size = cols[sp[i]].get(r), cols[sp[i] + 1].get(r)
        return SparseVector(0 if size is None else size, [] if idx is None else idx, v)
    return [tuple(value(i, r) for i in range(nf)) for r in range(batch.n_rows)]


class TFRecordDeserializer:
    """One record at a time, like the reference class; each call is one tfr_decode of a single frame (CRC
    check off: the payload never went through TFRecordReader here)."""

    def __init__(self, dataSchema: StructType, device: int = 0):
        self.schema = dataSchema
        self.device = device
        self._dec: Dict[int, _native.Decoder] = {}

    def _decoder(self, rt: int) -> "_native.Decoder":
        if rt not in self._dec:
            self._dec[rt] = _native.Decoder(self.schema, rt, self.device, flags=0)
        return self._dec[rt]

    def _one(self, payload: bytes, rt: int) -> tuple:
        frame = struct.pack("<QI", len(payload), 0) + bytes(payload) + b"\0\0\0\0"
        batch, _ = self._decoder(rt).decode(frame)
        try:
            batch.raise_if_error()
            return _rows_of(batch, self.schema if rt != 2 else None)[0]
        finally:
            batch.release()

    def deserializeByteArray(self, byteArray: bytes) -> tuple:
        return self._one(byteArray, 2)

    def deserializeExample(self, example: bytes) -> tuple:
        return self._one(example, 0)

    def deserializeSequenceExample(self, sequenceExample: bytes) -> tuple:
        return self._one(sequenceExample, 1)

    def close(self):
        for d in self._dec.values():
            d.close()
        self._dec = {}


class TFRecordSerializer:
    """Constructor validates the types like the reference's (featureConverters are built eagerly,
    M/TFRecordSerializer.scala:14 -> RuntimeException for unsupported types)."""

    def __init__(self, dataSchema: StructType, device: int = 0):
        self.schema = dataSchema
        self.device = device
        self._enc: Dict[int, _native.Encoder] = {}
        _native.Schema(dataSchema, 1).close()        # type validation only

    def _encoder(self, rt: int) -> "_native.Encoder":
        if rt not in self._enc:
            schema = byte_array_schema() if rt == 2 else self.schema
            self._enc[rt] = _native.Encoder(schema, rt, self.device)
        return self._enc[rt]

    def _one(self, row: Sequence, rt: int) -> bytes:
        schema = byte_array_schema() if rt == 2 else self.schema
        framed = self._encoder(rt).encode(columns_from_rows(schema, [tuple(row)], rt))
        return framed[12:-4]

    def serializeByteArray(self, row: Sequence) -> bytes:
        return self._one(row, 2)

    def serializeExample(self, row: Sequence) -> bytes:
        return self._one(row, 0)

    def serializeSequenceExample(self, row: Sequence) -> bytes:
        return self._one(row, 1)

    def close(self):
        for e in self._enc.values():
            e.close()
        self._enc = {}


class PartitionedFile:
    def __init__(self, filePath: str, start: int = 0, length: Optional[int] = None):
        self.filePath = filePath
        self.start = start
        self.length = os.path.getsize(filePath) if length is None else length

    def toPath(self):
        return self.filePath


def _stream_blocks(f, remaining: int, block: int, stage, process):
    """The block loop shared by readFile and inferSchema: reads `f` in blocks of about `block` bytes into stage(nbytes) (a
    writable uint8 array), calls process(buffer, nbytes, is_final) -> consumed bytes and carries the unconsumed tail (a
    partial record) into the next block.  Yields after every block so that the caller can drain rows in between."""
    carry = b""
    while True:
        want = min(max(block - len(carry), block // 2), remaining)   # a carried record larger than the block still makes progress
        chunk = f.read(want) if want > 0 else b""
        remaining -= len(chunk)
        final = remaining == 0 or len(chunk) < want
        nbytes = len(carry) + len(chunk)
        st = stage(max(nbytes, 1))
        if carry:
            st[: len(carry)] = np.frombuffer(carry, dtype=np.uint8)
        if chunk:
            st[len(carry): nbytes] = np.frombuffer(chunk, dtype=np.uint8)
        used = process(st, nbytes, final)
        yield
        carry = st[used:nbytes].tobytes()
        if final:
            return


class TFRecordFileReader:
    BLOCK_BYTES = 256 << 20

    @staticmethod
    def readFile(conf, options: Dict[str, str], file: PartitionedFile, schema: StructType, device: int = 0,
                 block_bytes: Optional[int] = None, dataSchema: Optional[StructType] = None) -> Iterator[tuple]:
        """Stages the file in blocks into the decoder's pinned staging slots and decodes each block on the GPU
        (tfr_decode_submit); where a block ends -- the carry into the next one -- is known as soon as its frame index has
        run (tfr_batch_consumed), so block k+1 is read and submitted while block k decodes and block k-1's rows are
        handed out.  Rows before a bad record are yielded, then the exception the reference would throw is raised.
        With options["mode"] = "DROPMALFORMED" a failing record is skipped instead (a framing error still raises), and
        the dropped records of each block are logged once, with the file offset of the first.  With "PERMISSIVE" it is a
        row of nulls, its payload in the corrupt-record column when `schema` holds it, and logged the same way.  With
        resyncFraming = "true" as well, a framing error does not raise: the bytes up to the next verified record are a lost
        region, dropped or read as one corrupt row, and each is logged with its file offset and length.
        `dataSchema` (default: `schema`) is the file's schema, which PERMISSIVE needs the corrupt-record column in.
        A LongType field of `schema` named _tmp_metadata_row_index or _tmp_metadata_record_offset (Spark's temporary
        metadata columns) holds each row's entry index in the file or the file offset of its entry (in the decompressed
        stream for a compressed file), filled on the GPU.  ByteArray rows are byteArray, then those fields."""
        rt = _record_type(options)
        vf = _vector_format(options)
        flags, corrupt = _read_mode(options, schema if dataSchema is None else dataSchema, schema)
        block = block_bytes or TFRecordFileReader.BLOCK_BYTES
        dec = _native.Decoder(_decoder_schema(schema), rt, device, flags, corrupt_field=corrupt, vector_format=vf)

        def gen():
            todo = []
            try:
                compressed = _codec_of_path(file.toPath()) is not None
                with _open_read(file.toPath()) as f:
                    if not compressed:
                        f.seek(file.start)
                    remaining = (1 << 62) if compressed else file.length          # a compressed file is read to its end
                    n_slots = dec.num_staging_slots()
                    turn = [0]
                    pos = [0 if compressed else file.start]     # where the next block starts in the (decompressed) file
                    entries = [0]                               # and the entries in front of it (the file is read whole)

                    def stage(nbytes):
                        st = dec.staging_slot(turn[0] % n_slots, nbytes)
                        turn[0] += 1
                        return st

                    def process(st, nbytes, final):
                        batch = dec.submit(st, is_final=final, nbytes=nbytes, first_entry=entries[0], first_offset=pos[0])
                        todo.append((batch, pos[0]))
                        used, n = batch.extent()
                        pos[0] += used
                        entries[0] += n
                        return used

                    def drain(batch, block_pos):
                        try:
                            for row in _rows_of(batch, schema if rt != 2 else None, vf):
                                yield row
                            if flags & (TFR_F_DROP_MALFORMED | TFR_F_PERMISSIVE):
                                dropped = batch.dropped()
                                if flags & TFR_F_RESYNC:
                                    for _, off, nb, code, _ in batch.dropped_spans():
                                        if code in _cabi.FRAMING_ERRORS:
                                            _LOG.warning("%s: %s %d bytes at file offset %d (%s); reading goes on at the next "
                                                         "verified record", file.toPath(),
                                                         "read as a corrupt row" if flags & TFR_F_PERMISSIVE else "lost", nb,
                                                         block_pos + off, _cabi.STATUS_NAMES.get(code, code))
                                    dropped = [e for e in dropped if e[2] not in _cabi.FRAMING_ERRORS]
                                if dropped:
                                    _LOG.warning("%s: %s %d malformed record(s) of the block at offset %d; the first at "
                                                 "file offset %d (%s)", file.toPath(),
                                                 "read as corrupt rows" if flags & TFR_F_PERMISSIVE else "dropped", len(dropped),
                                                 block_pos, block_pos + dropped[0][1], _cabi.STATUS_NAMES.get(dropped[0][2], dropped[0][2]))
                            batch.raise_if_error()
                        finally:
                            batch.release()

                    for _ in _stream_blocks(f, remaining, block, stage, process):
                        while len(todo) > 1:                 # the block before the one just submitted
                            yield from drain(*todo.pop(0))
                    while todo:
                        yield from drain(*todo.pop(0))
            finally:
                for batch, _ in todo:
                    batch.release()
                dec.close()

        return gen()


def _row_bytes(row, sparse: bool = False) -> int:
    """rough size of a buffered row's values (what decides when the writer flushes); `sparse`: vectors are written sparse"""
    n = 0
    for v in row:
        if v is None:
            continue
        if isinstance(v, (bytes, bytearray, str)):
            n += len(v) + 8
        elif isinstance(v, (DenseVector, SparseVector)):
            n += (12 * len(v.values) + 24) if sparse else (8 * v.size + 8)     # written as toSparse, or dense (toArray)
        elif isinstance(v, (list, tuple)):
            n += 8 + sum((len(x) + 8) if isinstance(x, (bytes, bytearray, str)) else (8 * len(x) + 8 if isinstance(x, (list, tuple)) else 8) for x in v)
        else:
            n += 8
    return n + 16


class TFRecordOutputWriter:
    FLUSH_ROWS = 1 << 16
    FLUSH_BYTES = 256 << 20        # large rows (images, long byte strings) flush by size: one tfr_encode call frames < 2 GiB

    def __init__(self, path: str, options: Dict[str, str], dataSchema: StructType, context=None, device: int = 0):
        self.path = path
        self.recordType = _record_type(options)                 # validated up front; the reference throws at the first write
        self.schema = byte_array_schema() if self.recordType == 2 else dataSchema
        self.vectorFormat = _vector_format(options)
        self._enc = _native.Encoder(self.schema, self.recordType, device, vector_format=self.vectorFormat)
        self._rows: List[tuple] = []
        self._bytes = 0
        self._out = _open_write(path, _codec_name((options or {}).get("codec", "")))   # CodecStreams.createOutputStream (:19)

    def write(self, row: Sequence) -> None:
        row = tuple(row)
        self._rows.append(row)
        self._bytes += _row_bytes(row, self.vectorFormat == "sparse")
        if len(self._rows) >= self.FLUSH_ROWS or self._bytes >= self.FLUSH_BYTES:
            self._flush()

    def _encode_rows(self, rows: List[tuple]) -> None:
        try:
            self._out.write(self._enc.encode(columns_from_rows(self.schema, rows, self.recordType, self.vectorFormat)))
        except _native.TfrError as e:
            if e.code != A_TFR_E_BATCH_TOO_LARGE or len(rows) < 2:
                raise
            half = len(rows) // 2                                # the size estimate was too low: frame the rows in two calls
            self._encode_rows(rows[:half])
            self._encode_rows(rows[half:])

    def _flush(self):
        if self._rows:
            rows, self._rows, self._bytes = self._rows, [], 0
            self._encode_rows(rows)

    def close(self) -> None:
        try:
            self._flush()
        finally:
            self._out.close()
            self._enc.close()


class DefaultSource:
    """The FileFormat surface that stays (M/DefaultSource.scala:23-143): names and meanings only."""

    def shortName(self) -> str:
        return "tfrecord"

    def isSplitable(self, *a, **k) -> bool:
        return False                                             # :26-29; splitting happens inside the native side

    def metadataSchemaFields(self) -> List[Tuple[str, str, "LongType"]]:
        """The generated metadata fields this source fills, as FileFormat.metadataSchemaFields lists them (Spark 3.4 / 3.5:
        FileSourceGeneratedMetadataStructField(name, temporary column name, LongType, nullable = false)) on top of Spark's
        file-constant ones, which Spark appends itself: (name, temporary column, type).  _metadata.row_index is the row's
        entry index in its file, _metadata.record_offset the file offset of its entry; readFile fills the temporary columns."""
        return [(ROW_INDEX, ROW_INDEX_TEMPORARY_COLUMN_NAME, LongType()),
                (RECORD_OFFSET, RECORD_OFFSET_TEMPORARY_COLUMN_NAME, LongType())]

    def inferSchema(self, options: Dict[str, str], files: Sequence[str], device: int = 0, dist=None):
        """M/DefaultSource.scala:31-39,48-70: the first non-empty file is scanned (the reference scans it twice);
        ByteArray has the fixed one-column schema.  With `dist`, every rank scans its shard of the files and the maps
        are merged with one all-reduce (sharding.allreduce_schema).
        options["mode"] as the reader takes it: FAILFAST (default) fails on the first failing record.  DROPMALFORMED and
        PERMISSIVE skip failing records (framing errors still fail, unless resyncFraming is "true": then the bytes up to
        the next verified record are skipped, each such region logged with its file offset), logging them once per file, and without `dist` take
        the first file whose records give any name (the reference's collectFirst(hasSchema), M/DefaultSource.scala:36-38),
        since a file of skipped records only would give an empty schema.  PERMISSIVE ignores features named by
        columnNameOfCorruptRecord and always ends the schema with that column (nullable BinaryType), so that the schema
        reads the files back under the options it was inferred with (buildReader refuses PERMISSIVE without it)."""
        from .sharding import allreduce_schema, codes_to_struct, shard_lpt
        mode, flags = _mode_flags(options)
        rt = _record_type(options)
        if rt == 2:
            return byte_array_schema()
        corrupt = _corrupt_column_name(options) if mode == "PERMISSIVE" else None
        distributed = dist is not None and dist.is_initialized()
        todo = [f for f in files if os.path.getsize(f) > 0]
        if distributed:
            mine = shard_lpt([os.path.getsize(f) for f in todo], dist.get_world_size())[dist.get_rank()]
            todo = [todo[i] for i in mine]
        elif mode == "FAILFAST":
            todo = todo[:1]
        inf = _native.Infer(rt, device, flags, corrupt)
        block = TFRecordFileReader.BLOCK_BYTES
        buf = [np.empty(0, dtype=np.uint8)]

        def stage(nbytes):
            if len(buf[0]) < nbytes:
                buf[0] = np.empty(nbytes + nbytes // 8, dtype=np.uint8)
            return buf[0]

        try:
            for f in todo:                       # streamed in blocks like readFile: files of any size, no whole-file copy
                pos, skipped = [0], []           # where the next block starts in the (decompressed) file; (file offset, code)

                def process(st, nb, final):
                    used = inf.update_block(st, final, nb)
                    skipped.extend((pos[0] + off, code) for _, off, code, _ in inf.skipped())
                    pos[0] += used
                    return used

                with _open_read(f) as fh:
                    remaining = (1 << 62) if _codec_of_path(f) is not None else os.path.getsize(f)
                    for _ in _stream_blocks(fh, remaining, block, stage, process):
                        pass
                if flags & TFR_F_RESYNC:
                    for off, code in skipped:
                        if code in _cabi.FRAMING_ERRORS:
                            _LOG.warning("%s: schema inference skipped the bytes from file offset %d to the next verified record (%s)",
                                         f, off, _cabi.STATUS_NAMES.get(code, code))
                    skipped = [e for e in skipped if e[1] not in _cabi.FRAMING_ERRORS]
                if skipped:
                    _LOG.warning("%s: schema inference skipped %d malformed record(s); the first at file offset %d (%s)", f,
                                 len(skipped), skipped[0][0], _cabi.STATUS_NAMES.get(skipped[0][1], skipped[0][1]))
                if mode != "FAILFAST" and not distributed and inf.result():
                    break                        # the first file whose kept records give a name
            local = inf.result()
        finally:
            inf.close()
        schema = codes_to_struct(allreduce_schema(local, dist, f"cuda:{device}" if distributed and dist.get_backend() == "nccl" else None))
        if corrupt is not None:
            schema = StructType(list(schema.fields) + [StructField(corrupt, BinaryType(), True)])
        return schema

    def buildReader(self, dataSchema: StructType, requiredSchema: StructType, options: Dict[str, str], device: int = 0):
        """-> PartitionedFile => Iterator[row] (filters are accepted and ignored, :123).  options["mode"]: FAILFAST (default),
        DROPMALFORMED, or PERMISSIVE when `dataSchema` holds the corrupt-record column, checked here, before any file is read."""
        _read_mode(options, dataSchema, requiredSchema)
        _vector_format(options)
        return lambda file: TFRecordFileReader.readFile(None, options, file, requiredSchema, device, dataSchema=dataSchema)

    def prepareWrite(self, options: Dict[str, str], dataSchema: StructType):
        codec = _codec_name((options or {}).get("codec", ""))             # :94-102: the option turns output compression on
        _vector_format(options)

        class _Factory:
            def newInstance(self_inner, path, schema, context=None):
                return TFRecordOutputWriter(path, options, schema, context)

            def getFileExtension(self_inner, context=None):                 # :110-112
                return ".tfrecord" + (_CODECS[codec][0] if codec else "")

        return _Factory()

    # convenience used by the tests: spark.read.format("tfrecord").schema(s).load(p) / df.write...save(p)
    def load(self, path: str, schema: StructType, options: Optional[Dict[str, str]] = None, device: int = 0) -> List[tuple]:
        files = [path] if os.path.isfile(path) else sorted(os.path.join(path, f) for f in os.listdir(path)
                                                           if not f.startswith(("_", ".")))
        reader = self.buildReader(schema, schema, options or {}, device)
        rows: List[tuple] = []
        for f in files:
            rows.extend(reader(PartitionedFile(f)))
        return rows

    def save(self, path: str, schema: StructType, rows: Sequence[Sequence], options: Optional[Dict[str, str]] = None) -> None:
        os.makedirs(path, exist_ok=True)
        factory = self.prepareWrite(options or {}, schema)
        w = factory.newInstance(os.path.join(path, "part-00000" + factory.getFileExtension()), schema)
        for r in rows:
            w.write(r)
        w.close()
        open(os.path.join(path, "_SUCCESS"), "wb").close()
