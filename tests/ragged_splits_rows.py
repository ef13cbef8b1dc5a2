"""Ragged fields stored with row splits (include/tfrgpu.h, RAGGED, Row splits) restated on top of tests/ragged_rows.py and
oracle/pyref -- test infrastructure.

Under nestedArrayFormat=ragged with raggedPartition=rowSplits an Example field x: ArrayType(ArrayType(T)) is the plain features
x_values (as with row lengths) and x_row_splits (ArrayType(LongType), nullable, appended after every field in the lengths
part's place): k + 1 entries 0, l0, l0+l1, .. for a row of k inner lists.  Reading parses the lowered schema by every existing
rule and then raises the two parts back into x, or fails the record with TFR_E_BAD_NESTING at x."""
from __future__ import annotations

from itertools import accumulate
from typing import Optional, Sequence, Tuple

import ragged_rows as RR
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import ArrayType, LongType, StructField, StructType

ragged_fields = RR.ragged_fields


def lowered_schema(schema: StructType) -> StructType:
    low = RR.lowered_schema(schema)
    n = len(schema.fields)
    return StructType(list(low.fields[:n]) + [StructField(schema.fields[i].name + A.TFR_RAGGED_ROW_SPLITS_SUFFIX, ArrayType(LongType()), True)
                                              for i in ragged_fields(schema)])


def splits(lengths: Sequence[int]) -> list:
    """the row splits of inner lists of these lengths: 0 and the running sums"""
    return [0] + list(accumulate(lengths))


def lower_row(schema: StructType, row: Sequence) -> tuple:
    """a row of `schema` as a row of lowered_schema(schema): x flattened in its place, its row splits appended"""
    low = RR.lower_row(schema, row)
    n = len(schema.fields)
    return low[:n] + tuple(None if lens is None else splits(lens) for lens in low[n:])


def encode(schema: StructType, rows: Sequence[Sequence]) -> bytes:
    """the framed Example records the writer produces for `rows`"""
    low = lowered_schema(schema)
    return b"".join(pyref.frame(pyref.serialize_example_bytes(low, lower_row(schema, r))) for r in rows)


def raise_row(schema: StructType, lowered: Sequence) -> Tuple[Optional[tuple], Optional[int]]:
    """a row read by the lowered schema's rules as a row of `schema`: (row, None), or (None, x) when ragged field x's parts
    disagree -- exactly one present, or splits that are empty, do not start at 0, decrease or do not end at the number of
    values (the first such x)"""
    n = len(schema.fields)
    out = list(lowered[:n])
    for k, i in enumerate(ragged_fields(schema)):
        vals, spl = lowered[i], lowered[n + k]
        if vals is None and spl is None:
            continue
        if (vals is None or spl is None or not spl or spl[0] != 0 or any(b < a for a, b in zip(spl, spl[1:]))
                or spl[-1] != len(vals)):
            return None, i
        out[i] = [list(vals[a:b]) for a, b in zip(spl, spl[1:])]
    return tuple(out), None


def read(schema: StructType, payload: bytes) -> Tuple[Optional[tuple], Optional[Tuple[int, int]]]:
    """(row, None) or (None, (TFR_E_* code, reported field)) for one Example payload read with raggedPartition=rowSplits.  An
    error of the lowered parse comes first (a splits part's at its ragged field); the consistency check last."""
    n = len(schema.fields)
    rg = ragged_fields(schema)
    row, err = RR.parse_lowered(lowered_schema(schema), payload)
    if err is not None:
        return None, (err[0], rg[err[1] - n] if err[1] >= n else err[1])
    r, bad = raise_row(schema, row)
    return (r, None) if bad is None else (None, (A.TFR_E_BAD_NESTING, bad))
