"""Sparse-format VectorUDT fields (include/tfrgpu.h, SPARSE VECTORS) as Spark UnsafeRow bytes and as their lowered twin -- test
infrastructure next to tests/vector_rows.py, whose struct writer it reuses.

A sparse vector `v` is the three ordinary fields v_values (ArrayType(DoubleType), in v's place), v_indices (ArrayType(IntegerType))
and v_size (IntegerType), the two parts appended after every field (sqltypes.lowered_schema): the twin schema.  On write its
parts are those of v.toSparse; on read the UnsafeRow slot holds the nested row of VectorUDT.serialize(SparseVector(size, indices,
values)): type 0, size, indices, values, where a null size or indices is a null bit and a zero slot and the array behind it
moves up (vector_rows.struct_bytes lays out exactly that)."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

import vector_rows as V
from spark_tfrecord_b200.sqltypes import (StructType, VectorUDT, lowered_schema, sparse_parts, sparse_vector_fields)


class SparseParts:
    """a decoded sparse vector given as its three parts as they are (None: that part is null)"""

    def __init__(self, size: Optional[int], indices: Optional[Sequence[int]], values: Sequence[float]):
        self.size, self.indices, self.values = size, indices, values


def sparse_struct(size: Optional[int], indices: Optional[Sequence[int]], values: Sequence[float]) -> bytes:
    """the nested row the reader writes for a sparse vector's parts"""
    return V.struct_bytes(0, size, None if indices is None else V.int_array(indices), V.double_array(values))


def unsafe_rows(schema: StructType, rows: Sequence[Sequence]):
    """vector_rows.unsafe_rows, with SparseParts values of VectorUDT fields written as the reader's sparse nested row"""
    conv = [tuple(V.RawVector(sparse_struct(v.size, v.indices, v.values)) if isinstance(v, SparseParts) else v for v in row)
            for row in rows]
    return V.unsafe_rows(schema, conv)


def twin_rows(schema: StructType, rows: Sequence[Sequence]) -> List[tuple]:
    """rows of `schema` (DenseVector / SparseVector values) as rows of its sparse-format twin, lowered_schema(schema, "sparse"):
    each vector's toSparse values in its place, then (indices, size) of every vector in field order"""
    sp = sparse_vector_fields(schema, "sparse")
    out = []
    for row in rows:
        parts = [sparse_parts(row[i]) for i in sp]
        out.append(tuple(parts[sp.index(i)][1] if i in sp else v for i, v in enumerate(row)) +
                   tuple(x for p in parts for x in (p[0], p[2])))
    return out


def twin_schema(schema: StructType) -> StructType:
    return lowered_schema(schema, "sparse")


def parts_of_columns(cols, schema: StructType, r: int) -> tuple:
    """row r of a sparse-format decode's columns as a row of `schema`: SparseParts for each VectorUDT field (None: null)"""
    nf = len(schema)
    sp = sparse_vector_fields(schema, "sparse")
    row = []
    for i in range(nf):
        v = cols[i].get(r)
        if i in sp and v is not None:
            k = nf + 2 * sp.index(i)
            v = SparseParts(cols[k + 1].get(r), cols[k].get(r), np.asarray(v, dtype=np.float64))
        row.append(v)
    return tuple(row)


def is_vector(f) -> bool:
    return isinstance(f.dataType, VectorUDT)
