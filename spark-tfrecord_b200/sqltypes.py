"""Spark SQL type mirror for the schema-facing part of the reference API.

The reference takes a Spark ``StructType`` everywhere (``new TFRecordDeserializer(schema)``
M/TFRecordFileReader.scala:44, ``new TFRecordSerializer(dataSchema)`` M/TFRecordOutputWriter.scala:24).
There is no Spark/JVM in this image, so the same names are provided as plain Python objects; they
lower to the C ABI's ``tfr_field`` (include/tfrgpu.h).  M/ = src/main/scala/com/linkedin/spark/datasources/tfrecord/
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence

import numpy as np

# tfr type ids (include/tfrgpu.h)
TFR_T_NULL, TFR_T_INT32, TFR_T_INT64, TFR_T_FLOAT32, TFR_T_FLOAT64, TFR_T_DECIMAL, TFR_T_STRING, TFR_T_BINARY = range(8)
TFR_T_ROW_INDEX, TFR_T_RECORD_OFFSET = 8, 9          # generated fields: read as LongType, never from a record
TFR_T_VECTOR = 10                                      # Spark ML's VectorUDT (include/tfrgpu.h, VECTORS)
TFR_T_SPARSE_VECTOR = 11                               # the same, as TF sparse features (include/tfrgpu.h, SPARSE VECTORS)
# the feature keys of a sparse vector `v`: v + suffix (TFR_SPARSE_*_SUFFIX of include/tfrgpu.h)
SPARSE_INDICES_SUFFIX, SPARSE_VALUES_SUFFIX, SPARSE_SIZE_SUFFIX = "_indices", "_values", "_size"
VECTOR_FORMATS = ("dense", "sparse")                   # the `vectorFormat` DataSource option; dense is the default
TFR_T_UNSUPPORTED = 99
TFR_RT_EXAMPLE, TFR_RT_SEQUENCE_EXAMPLE, TFR_RT_BYTE_ARRAY = range(3)

RECORD_TYPES = {"Example": TFR_RT_EXAMPLE, "SequenceExample": TFR_RT_SEQUENCE_EXAMPLE, "ByteArray": TFR_RT_BYTE_ARRAY}


class DataType:
    tfr_id = TFR_T_UNSUPPORTED

    def __eq__(self, other):
        return type(self) is type(other) and self.__dict__ == other.__dict__

    def __hash__(self):
        return hash(type(self).__name__)

    def __repr__(self):
        return type(self).__name__


class NullType(DataType):
    tfr_id = TFR_T_NULL


class IntegerType(DataType):
    tfr_id = TFR_T_INT32


class LongType(DataType):
    tfr_id = TFR_T_INT64


class FloatType(DataType):
    tfr_id = TFR_T_FLOAT32


class DoubleType(DataType):
    tfr_id = TFR_T_FLOAT64


class DecimalType(DataType):
    """Carried as float64 across the C ABI (``Decimal(f.toDouble)``, M/TFRecordDeserializer.scala:86-87);
    the JVM shim wraps the double in ``Decimal``."""
    tfr_id = TFR_T_DECIMAL


class StringType(DataType):
    tfr_id = TFR_T_STRING


class BinaryType(DataType):
    tfr_id = TFR_T_BINARY


class RowIndexType(DataType):
    """A generated LongType field: the row's entry index in its file (include/tfrgpu.h, POSITIONS).  Not a Spark type: the
    reader puts it in place of the LongType of Spark's temporary metadata column (io.readFile)."""
    tfr_id = TFR_T_ROW_INDEX


class RecordOffsetType(DataType):
    """A generated LongType field: the file offset of the row's entry (include/tfrgpu.h, POSITIONS)."""
    tfr_id = TFR_T_RECORD_OFFSET


class VectorUDT(DataType):
    """Spark ML's ``org.apache.spark.ml.linalg.VectorUDT`` (``org.apache.spark.mllib.linalg.VectorUDT`` has the same sqlType and
    maps to it too).  Read as a dense vector of what an ArrayType(DoubleType) field reads; written as the FloatList of
    ``toArray`` (include/tfrgpu.h, VECTORS).  Only as a top-level field: ArrayType(VectorUDT) is refused."""
    tfr_id = TFR_T_VECTOR
    CLASS_NAMES = ("org.apache.spark.ml.linalg.VectorUDT", "org.apache.spark.mllib.linalg.VectorUDT")

    @staticmethod
    def sqlType() -> str:
        return "struct<type:tinyint,size:int,indices:array<int>,values:array<double>>"


class DenseVector:
    """Spark ML's DenseVector: the value type of a VectorUDT field as the reader returns it."""

    def __init__(self, values):
        self.values = np.asarray(values, dtype=np.float64).reshape(-1)

    @property
    def size(self) -> int:
        return len(self.values)

    def toArray(self) -> np.ndarray:
        return self.values

    def toSparse(self) -> "SparseVector":
        return _to_sparse(self.size, np.arange(self.size, dtype=np.int32), self.values)

    def __eq__(self, other):
        return isinstance(other, (DenseVector, SparseVector)) and np.array_equal(self.toArray(), other.toArray())

    def __len__(self):
        return self.size

    def __repr__(self):
        return f"DenseVector({self.values.tolist()!r})"


class SparseVector:
    """Spark ML's SparseVector, with its constructor's checks: size >= 0, as many indices as values, indices strictly
    increasing inside [0, size)."""

    def __init__(self, size: int, indices, values):
        self.size = int(size)
        self.indices = np.asarray(indices, dtype=np.int32).reshape(-1)
        self.values = np.asarray(values, dtype=np.float64).reshape(-1)
        if self.size < 0:
            raise ValueError(f"the size of a sparse vector must be no less than 0, not {self.size}")
        if len(self.indices) != len(self.values):
            raise ValueError(f"{len(self.indices)} indices and {len(self.values)} values")
        if len(self.indices) and (self.indices[0] < 0 or self.indices[-1] >= self.size or np.any(np.diff(self.indices) <= 0)):
            raise ValueError(f"indices must be strictly increasing and inside [0, {self.size})")

    def toArray(self) -> np.ndarray:
        out = np.zeros(self.size, dtype=np.float64)
        out[self.indices] = self.values
        return out

    def toSparse(self) -> "SparseVector":
        return _to_sparse(self.size, self.indices, self.values)

    def __eq__(self, other):
        return isinstance(other, (DenseVector, SparseVector)) and np.array_equal(self.toArray(), other.toArray())

    def __len__(self):
        return self.size

    def __repr__(self):
        return f"SparseVector({self.size}, {self.indices.tolist()!r}, {self.values.tolist()!r})"


def _to_sparse(size: int, indices: np.ndarray, values: np.ndarray) -> SparseVector:
    """Vector.toSparse: the entries whose double is != 0.0 (-0.0 and stored zeros dropped, NaN kept), in index order."""
    keep = values != 0.0
    return SparseVector(size, indices[keep], values[keep])


class TimestampType(DataType):
    """Exists only so the reference's "unsupported data type" tests can be restated."""


class BooleanType(DataType):
    pass


class ArrayType(DataType):
    def __init__(self, elementType: DataType, containsNull: bool = True):
        self.elementType = elementType
        self.containsNull = containsNull

    def __eq__(self, other):
        return isinstance(other, ArrayType) and self.elementType == other.elementType

    def __hash__(self):
        return hash(("array", self.elementType))

    def __repr__(self):
        return f"ArrayType({self.elementType!r})"


@dataclass
class StructField:
    name: str
    dataType: DataType
    nullable: bool = True


class StructType:
    def __init__(self, fields: Sequence[StructField] = ()):
        self.fields: List[StructField] = list(fields)

    def __iter__(self):
        return iter(self.fields)

    def __len__(self):
        return len(self.fields)

    def __getitem__(self, i):
        return self.fields[i]

    def add(self, name, dataType, nullable=True):
        self.fields.append(StructField(name, dataType, nullable))
        return self

    @property
    def names(self):
        return [f.name for f in self.fields]

    def __repr__(self):
        return "StructType(%s)" % ", ".join(f"{f.name}:{f.dataType!r}{'' if f.nullable else ' NOT NULL'}" for f in self.fields)


def check_vector_format(vector_format: str) -> str:
    """the `vectorFormat` option's value, refused (ValueError naming the option) unless it is one of VECTOR_FORMATS"""
    if vector_format not in VECTOR_FORMATS:
        raise ValueError(f"vectorFormat must be one of {', '.join(VECTOR_FORMATS)}, not {vector_format!r}")
    return vector_format


def lower_type(dt: DataType, vector_format: str = "dense"):
    """DataType -> (elem_type_id, depth).  Anything the reference rejects lowers to
    (TFR_T_UNSUPPORTED, depth) and is refused by tfr_schema_create; so is ArrayType(VectorUDT), (TFR_T_VECTOR, depth > 0).
    A VectorUDT is TFR_T_VECTOR, or TFR_T_SPARSE_VECTOR with vector_format="sparse"."""
    check_vector_format(vector_format)
    depth = 0
    while isinstance(dt, ArrayType):
        depth += 1
        dt = dt.elementType
    if dt.tfr_id == TFR_T_VECTOR and vector_format == "sparse":
        return TFR_T_SPARSE_VECTOR, depth
    return dt.tfr_id, depth


def sparse_vector_fields(schema: StructType, vector_format: str = "dense") -> List[int]:
    """the indexes of the top-level fields that are sparse vectors under vector_format, in field order"""
    check_vector_format(vector_format)
    return [i for i, f in enumerate(schema) if vector_format == "sparse" and isinstance(f.dataType, VectorUDT)]


def lowered_schema(schema: StructType, vector_format: str = "dense") -> StructType:
    """The schema every kernel sees (include/tfrgpu.h, SPARSE VECTORS): a sparse vector `v` is its values field
    v_values: ArrayType(DoubleType) in its place, with its nullability, and the nullable fields v_indices: ArrayType(IntegerType)
    and v_size: IntegerType appended after all the fields, in field order.  Its columns are the decoder's and the encoder's."""
    sp = set(sparse_vector_fields(schema, vector_format))
    out = [StructField(f.name + SPARSE_VALUES_SUFFIX, ArrayType(DoubleType()), f.nullable) if i in sp else f
           for i, f in enumerate(schema)]
    for i in sorted(sp):
        nm = schema[i].name
        out.append(StructField(nm + SPARSE_INDICES_SUFFIX, ArrayType(IntegerType()), True))
        out.append(StructField(nm + SPARSE_SIZE_SUFFIX, IntegerType(), True))
    return StructType(out)


def sparse_parts(v):
    """A vector (DenseVector or SparseVector, or None) -> the values of its three lowered fields, (indices, values, size) of
    v.toSparse, or (None, None, None) for a null vector."""
    if v is None:
        return None, None, None
    s = v.toSparse()
    return s.indices.tolist(), s.values.tolist(), int(s.size)


# TensorFlowInferSchema.getSchemaForByteArray (M/TensorFlowInferSchema.scala:60-64)
def byte_array_schema() -> StructType:
    return StructType([StructField("byteArray", BinaryType())])
