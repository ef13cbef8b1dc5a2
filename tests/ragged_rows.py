"""Ragged fields (include/tfrgpu.h, RAGGED) restated on top of the plain lowered schema -- test infrastructure next to
tests/sparse_vector_rows.py.

Under nestedArrayFormat=ragged an Example field x: ArrayType(ArrayType(T)) is the two plain features x_values (ArrayType(T), in
x's place and with x's nullability) and x_row_lengths (ArrayType(LongType), nullable, appended after every field).  Writing
lowers a row; reading parses the lowered schema by every existing rule (oracle/pyref) and then raises the two parts back into
x, or fails the record with TFR_E_BAD_NESTING at x."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import ArrayType, LongType, StructField, StructType


def ragged_fields(schema: StructType) -> List[int]:
    return [i for i, f in enumerate(schema.fields)
            if isinstance(f.dataType, ArrayType) and isinstance(f.dataType.elementType, ArrayType)]


def lowered_schema(schema: StructType) -> StructType:
    rg = ragged_fields(schema)
    fields = [StructField(f.name + A.TFR_RAGGED_VALUES_SUFFIX, f.dataType.elementType, f.nullable) if i in rg else f
              for i, f in enumerate(schema.fields)]
    fields += [StructField(schema.fields[i].name + A.TFR_RAGGED_ROW_LENGTHS_SUFFIX, ArrayType(LongType()), True) for i in rg]
    return StructType(fields)


def lower_row(schema: StructType, row: Sequence) -> tuple:
    """a row of `schema` as a row of lowered_schema(schema): x flattened in its place, its inner lengths appended"""
    rg = ragged_fields(schema)
    flat = tuple(None if (i in rg and v is None) else [e for inner in v for e in inner] if i in rg else v
                 for i, v in enumerate(row))
    return flat + tuple(None if row[i] is None else [len(inner) for inner in row[i]] for i in rg)


def encode(schema: StructType, rows: Sequence[Sequence]) -> bytes:
    """the framed Example records the writer produces for `rows`"""
    low = lowered_schema(schema)
    return b"".join(pyref.frame(pyref.serialize_example_bytes(low, lower_row(schema, r))) for r in rows)


def raise_row(schema: StructType, lowered: Sequence) -> Tuple[Optional[tuple], Optional[int]]:
    """a row read by the lowered schema's rules as a row of `schema`: (row, None), or (None, x) when ragged field x's parts
    disagree -- exactly one present, a negative length, or lengths that do not sum to the number of values (the first such x)"""
    rg = ragged_fields(schema)
    n = len(schema.fields)
    out = list(lowered[:n])
    for k, i in enumerate(rg):
        vals, lens = lowered[i], lowered[n + k]
        if vals is None and lens is None:
            continue
        if vals is None or lens is None or any(l < 0 for l in lens) or sum(lens) != len(vals):
            return None, i
        it, nested = 0, []
        for l in lens:
            nested.append(list(vals[it:it + l]))
            it += l
        out[i] = nested
    return tuple(out), None


def parse_lowered(low: StructType, payload: bytes, unkeyed=()) -> Tuple[Optional[list], Optional[Tuple[int, int]]]:
    """one Example payload parsed by the plain rules of every field of `low` (oracle/pyref), field by field in order: (values,
    None), or (None, (TFR_E_* code, lowered field)) at the first field that fails.  A field in `unkeyed` is no feature's (a
    generated field, the corrupt-record column): it is read as None and never fails."""
    ex = pyref.Example()
    try:
        ex.ParseFromString(payload)
    except Exception:
        return None, (A.TFR_E_MALFORMED_PROTO, -1)
    row = []
    for f_i, f in enumerate(low.fields):
        if f_i in unkeyed:
            row.append(None)
            continue
        try:
            row.append(pyref.deserialize_example(StructType([f]), ex)[0])
        except pyref.RefError as e:
            code = {"NullPointerException": A.TFR_E_NULL_IN_NONNULL, "NoSuchElementException": A.TFR_E_EMPTY_SCALAR}.get(
                e.java_class, A.TFR_E_KIND_MISMATCH)
            return None, (code, f_i)
    return row, None


def read(schema: StructType, payload: bytes) -> Tuple[Optional[tuple], Optional[Tuple[int, int]]]:
    """(row, None) or (None, (TFR_E_* code, reported field)) for one Example payload read with nestedArrayFormat=ragged.  An
    error of the lowered parse comes first (a lengths part's at its ragged field); the consistency check last."""
    n = len(schema.fields)
    rg = ragged_fields(schema)
    row, err = parse_lowered(lowered_schema(schema), payload)
    if err is not None:
        return None, (err[0], rg[err[1] - n] if err[1] >= n else err[1])
    r, bad = raise_row(schema, row)
    return (r, None) if bad is None else (None, (A.TFR_E_BAD_NESTING, bad))
