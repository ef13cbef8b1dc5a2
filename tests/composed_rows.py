"""Every schema lowering at once, restated from the per-feature modules -- test infrastructure for schemas that combine dense
and sparse VectorUDT fields (include/tfrgpu.h, VECTORS, SPARSE VECTORS), ragged fields with row lengths or row splits
(RAGGED), extendedTypes=true fields (INT64 TYPES), the generated fields (POSITIONS) and a PERMISSIVE corrupt-record column.

The library lowers a caller's schema into plain fields, in this order (tfr_schema_create_ex):
  1. the caller's fields, each lowered in its place: a dense vector is ArrayType(DoubleType), a sparse vector its v_values
     part, a ragged x its x_values part (ArrayType(T)), an INT64 TYPES leaf a LongType leaf, a generated field a nullable
     LongType that no feature maps to, the corrupt-record column a BinaryType that no feature maps to;
  2. every sparse vector's v_indices and v_size, in field order;
  3. every ragged field's x_row_lengths (or x_row_splits), in field order.
A part reports errors at its owner: the vector or the ragged field it belongs to.

Rows of a caller's schema hold: ints for INT64 TYPES leaves (as their columns hold them: bool 0 / 1, days, microseconds),
DenseVector / SparseVector for vectors (a read gives DenseVector, or sparse_vector_rows.SparseParts in the sparse format),
nested lists for ragged fields, and ints for the generated fields.  Writing and reading go through oracle/pyref on the
lowered schema, each lowering by its own module: vector_rows, sparse_vector_rows, ragged_rows, ragged_splits_rows,
int64_types; the expected UnsafeRows through partition_rows' writer."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

import int64_types as I
import partition_rows as PR
import position_walk as PW
import ragged_rows as RR
import ragged_splits_rows as RS
import resync_walk as RW
import sparse_vector_rows as SP
import vector_rows as V
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import (SPARSE_INDICES_SUFFIX, SPARSE_SIZE_SUFFIX, SPARSE_VALUES_SUFFIX, ArrayType,
                                          BinaryType, DenseVector, DoubleType, FloatType, IntegerType, LongType,
                                          RecordOffsetType, RowIndexType, SparseVector, StringType, StructField, StructType,
                                          VectorUDT)


class Opts:
    """the reader's and writer's options: vectorFormat, nestedArrayFormat=ragged, raggedPartition=rowSplits,
    extendedTypes=true, and the corrupt-record column (the caller's field index; PERMISSIVE only)"""

    def __init__(self, vector_format: str = "dense", ragged: bool = False, row_splits: bool = False,
                 extended_types: bool = False, corrupt: Optional[int] = None):
        self.vector_format, self.ragged, self.row_splits = vector_format, ragged, row_splits
        self.extended_types, self.corrupt = extended_types, corrupt

    def native(self) -> dict:
        """the keyword arguments of _native.Decoder / Encoder"""
        return dict(vector_format=self.vector_format, ragged=self.ragged, row_splits=self.row_splits,
                    extended_types=self.extended_types)

    def __repr__(self):
        return (f"Opts({self.vector_format}, ragged={self.ragged}, splits={self.row_splits}, ext={self.extended_types}, "
                f"corrupt={self.corrupt})")


def generated(f) -> bool:
    return isinstance(f.dataType, (RowIndexType, RecordOffsetType))


def unkeyed(schema: StructType, opts: Opts) -> List[int]:
    """the caller's fields no feature maps to: the generated fields and the corrupt-record column"""
    return [i for i, f in enumerate(schema) if generated(f) or i == opts.corrupt]


def write_schema(schema: StructType, opts: Opts) -> StructType:
    """the schema a writer takes: the caller's without the generated fields and the corrupt-record column"""
    skip = set(unkeyed(schema, opts))
    return StructType([f for i, f in enumerate(schema) if i not in skip])


def _sparse(schema: StructType, opts: Opts) -> List[int]:
    return [i for i, f in enumerate(schema) if isinstance(f.dataType, VectorUDT) and opts.vector_format == "sparse"]


def _ragged(schema: StructType, opts: Opts) -> List[int]:
    return RR.ragged_fields(schema) if opts.ragged else []


def _i64(f, opts: Opts) -> int:
    return I.leaf_id(f.dataType) if opts.extended_types else 0


def lowered_schema(schema: StructType, opts: Opts) -> StructType:
    """the plain schema every parse and encode kernel sees, in the library's field order (see the module's docstring)"""
    sp, rg = _sparse(schema, opts), _ragged(schema, opts)
    out = []
    for i, f in enumerate(schema):
        if generated(f):
            out.append(StructField(f.name, LongType(), True))
        elif isinstance(f.dataType, VectorUDT):
            out.append(StructField(f.name + (SPARSE_VALUES_SUFFIX if i in sp else ""), ArrayType(DoubleType()), f.nullable))
        elif i in rg:
            out.append(StructField(f.name + A.TFR_RAGGED_VALUES_SUFFIX, I.long_type(f.dataType.elementType), f.nullable))
        else:
            out.append(StructField(f.name, I.long_type(f.dataType) if opts.extended_types else f.dataType, f.nullable))
    for i in sp:
        out += [StructField(schema[i].name + SPARSE_INDICES_SUFFIX, ArrayType(IntegerType()), True),
                StructField(schema[i].name + SPARSE_SIZE_SUFFIX, IntegerType(), True)]
    suffix = A.TFR_RAGGED_ROW_SPLITS_SUFFIX if opts.row_splits else A.TFR_RAGGED_ROW_LENGTHS_SUFFIX
    out += [StructField(schema[i].name + suffix, ArrayType(LongType()), True) for i in rg]
    return StructType(out)


def n_lowered(schema: StructType, opts: Opts) -> int:
    """the lowered field count: n + 2 per sparse vector + 1 per ragged field (the fast paths take at most 128)"""
    return len(schema) + 2 * len(_sparse(schema, opts)) + len(_ragged(schema, opts))


def n_narrowed(schema: StructType, opts: Opts) -> int:
    """the columns narrow_kernel and widen_kernel convert: INT64 TYPES fields but timestamps (NARROW_MAX per launch)"""
    return sum(1 for f in schema if _i64(f, opts) not in (0, A.TFR_T_TIMESTAMP))


def owner(schema: StructType, opts: Opts, lf: int) -> int:
    """the caller's field of lowered field lf"""
    n, sp, rg = len(schema), _sparse(schema, opts), _ragged(schema, opts)
    if lf < n:
        return lf
    return sp[(lf - n) // 2] if lf < n + 2 * len(sp) else rg[lf - n - 2 * len(sp)]


# ---- write ----
def lower_row(schema: StructType, row: Sequence, opts: Opts) -> tuple:
    """a row of the writer's schema as a row of its lowered schema"""
    (row,) = I.long_rows(schema, [row]) if opts.extended_types else (row,)
    n = len(schema)
    if opts.vector_format == "sparse":
        row = SP.twin_rows(schema, [row])[0]
    else:
        row = V.as_double_rows(schema, [row])[0]
    head, parts = row[:n], row[n:]
    if not opts.ragged:
        return tuple(head) + tuple(parts)
    rag = (RS if opts.row_splits else RR).lower_row(schema, head)
    return tuple(rag[:n]) + tuple(parts) + tuple(rag[n:])


def encode(schema: StructType, rows: Sequence[Sequence], opts: Opts) -> bytes:
    """the framed Example records the writer produces for `rows` of its schema"""
    low = lowered_schema(schema, opts)
    return b"".join(pyref.frame(pyref.serialize_example_bytes(low, lower_row(schema, r, opts))) for r in rows)


def to_py(schema: StructType, row: Sequence, opts: Opts) -> tuple:
    """a row's INT64 TYPES ints as the Python values the writer's columns take (bool, int, date, aware datetime)"""
    out = []
    for f, v in zip(schema, row):
        t = _i64(f, opts)
        out.append(_map(lambda x: A.int64_value(t, x), v) if t else v)
    return tuple(out)


def _map(fn, v):
    if v is None:
        return None
    if isinstance(v, list):
        return [_map(fn, e) for e in v]
    return fn(v)


# ---- read ----
def _narrow(t: int, v):
    """int64 values read by the LongType rule -> the narrow ints a read gives (int64_types.narrow, leaf by leaf)"""
    if v is None:
        return None
    if isinstance(v, list):
        return [_narrow(t, e) for e in v]
    return int(I.narrow(t, np.array([v], dtype=np.int64))[0])


def read(schema: StructType, payload: bytes, opts: Opts) -> Tuple[Optional[tuple], Optional[Tuple[int, int]]]:
    """(row, None) or (None, (TFR_E_* code, the owner's field)) for one Example payload.  The lowered parse's errors come
    first, in lowered field order; the ragged consistency check last.  Generated fields and the corrupt-record column are
    None in the row (they are not the record's)."""
    low = lowered_schema(schema, opts)
    n, sp = len(schema), _sparse(schema, opts)
    vals, err = RR.parse_lowered(low, payload, set(unkeyed(schema, opts)))
    if err is not None:
        return None, (err[0], err[1] if err[1] < 0 else owner(schema, opts, err[1]))
    head = list(vals[:n])
    if opts.ragged:
        raised, bad = (RS if opts.row_splits else RR).raise_row(schema, head + vals[n + 2 * len(sp):])
        if bad is not None:
            return None, (A.TFR_E_BAD_NESTING, bad)
        head = list(raised)
    out = []
    for i, f in enumerate(schema):
        v, t = head[i], _i64(f, opts)
        if isinstance(f.dataType, VectorUDT) and v is not None:
            if i in sp:
                k = n + 2 * sp.index(i)
                v = SP.SparseParts(vals[k + 1], vals[k], v)
            else:
                v = DenseVector(v)
        elif t:
            v = _narrow(t, v)
        out.append(v)
    return tuple(out), None


def column_row(schema: StructType, row: Sequence, opts: Opts) -> tuple:
    """a read row as the decoder's columns hold it: the caller's fields (a vector as its values), then every sparse vector's
    (indices, size)"""
    out, parts = [], []
    for i, (f, v) in enumerate(zip(schema, row)):
        if isinstance(f.dataType, VectorUDT):
            if i in _sparse(schema, opts):
                s = v if isinstance(v, SP.SparseParts) or v is None else SP.SparseParts(*_sparse_of(v))
                parts += [None, None] if s is None else [s.indices, s.size]
                v = None if s is None else s.values
            elif v is not None:
                v = v.toArray()
        out.append(v)
    return tuple(out) + tuple(parts)


def _sparse_of(v):
    ind, vals, size = SP.sparse_parts(v)
    return size, ind, vals


def canon(v):
    """a value in one form for exact comparison: floats as their float64 bits, strings as UTF-8 bytes, vectors and arrays
    as lists, INT64 TYPES objects as their column ints"""
    import datetime as dt
    if v is None:
        return None
    if isinstance(v, (DenseVector, SparseVector, SP.SparseParts)):
        s = v if isinstance(v, SP.SparseParts) else SP.SparseParts(*_sparse_of(v))
        return ("vec", canon(s.size), canon(s.indices), canon(s.values))
    if isinstance(v, np.ndarray):
        return [canon(x) for x in v.tolist()]
    if isinstance(v, (list, tuple)):
        return [canon(x) for x in v]
    if isinstance(v, (float, np.floating)):
        return ("f", int(np.array([v], dtype=np.float64).view(np.uint64)[0]))
    if isinstance(v, bool):
        return int(v)
    if isinstance(v, dt.datetime):
        return A.int64_leaf(A.TFR_T_TIMESTAMP, v)
    if isinstance(v, dt.date):
        return A.int64_leaf(A.TFR_T_DATE, v)
    if isinstance(v, np.integer):
        return int(v)
    if isinstance(v, str):                                  # (pyref reads a string as its UTF-8 bytes)
        return v.encode("utf-8")
    return v


def columns_rows(cols, n_rows: int) -> List[list]:
    """the decoder's host columns, row by row, in canon form"""
    return [[canon(c.get(r)) for c in cols] for r in range(n_rows)]


# ---- a block: the rows, errors and positions every mode gives ----
def payload_crc_ok(data: bytes, off: int, end: int) -> bool:
    return pyref.masked_crc32c(bytes(data[off + 12:end - 4])) == int.from_bytes(data[end - 4:end], "little")


class Expect:
    """what a decoder of `schema` in `mode` (PW.FAILFAST, DROPMALFORMED or PERMISSIVE; `resync`: TFR_F_RESYNC) gives for one
    final block: rows (read rows with the generated fields and the corrupt-record column filled), dropped
    [(entry, code, field)], error (code, row, field) or None"""

    def __init__(self, schema: StructType, opts: Opts, data: bytes, mode: str, resync: bool = False):
        data = bytes(data)
        ents, _ = PW.entries(data, True, resync)
        stop = 0 if resync else RW.chain(data, 0, True)[2]
        verdicts = []
        for e in ents:
            if e[0] == "region":
                verdicts.append((None, (e[3], -1)))
            elif not payload_crc_ok(data, e[1], e[2]):
                verdicts.append((None, (A.TFR_E_CRC_DATA, -1)))
            else:
                verdicts.append(read(schema, data[e[1] + 12:e[2] - 4], opts))
        bad = [k for k, v in enumerate(verdicts) if v[1] is not None]
        self.error, self.dropped = None, []
        if mode == PW.FAILFAST:
            keep = list(range(bad[0] if bad else len(ents)))
            if bad:
                self.error = (verdicts[bad[0]][1][0], bad[0], verdicts[bad[0]][1][1])
        else:
            self.dropped = [(k,) + verdicts[k][1] for k in bad]
            keep = list(range(len(ents))) if mode == PW.PERMISSIVE else [k for k in range(len(ents)) if k not in bad]
        if stop and self.error is None:
            self.error = (stop, len(ents), -1)
        gen = [i for i, f in enumerate(schema) if generated(f)]
        self.rows = []
        for k in keep:
            row, err = verdicts[k]
            row = list(row) if err is None else [None] * len(schema)
            if err is not None and opts.corrupt is not None:
                e = ents[k]
                row[opts.corrupt] = data[e[1]:e[2]] if e[0] == "region" else data[e[1] + 12:e[2] - 4]
            for i in gen:
                row[i] = k if isinstance(schema[i].dataType, RowIndexType) else ents[k][1]
            self.rows.append(tuple(row))


# ---- UnsafeRows ----
def write_field(opts: Opts):
    """partition_rows' per-field writer with the lowerings: a vector as its nested struct (vector_rows,
    sparse_vector_rows), an INT64 TYPES field at its narrow width (int64_types), anything else as oracle.unsaferow writes it"""
    def write(w, i, f, v):
        t = _i64(f, opts)
        if v is None:
            w.set_null(i)
        elif isinstance(v, V.RawVector):                     # a malformed struct, as it is
            w.var(i, v.data)
        elif isinstance(f.dataType, VectorUDT):
            w.var(i, SP.sparse_struct(v.size, v.indices, v.values) if isinstance(v, SP.SparseParts) else V.vector_struct(v))
        elif t and not isinstance(f.dataType, ArrayType):
            w.slot(i, int(v) & ((1 << (8 * I._width(t))) - 1))
        elif t:
            depth, dt = 0, f.dataType
            while isinstance(dt, ArrayType):
                depth, dt = depth + 1, dt.elementType
            w.var(i, I.unsafe_array(t, depth, v))
        elif generated(f):
            w.slot(i, int(v))
        else:
            PR.write_data_field(w, i, f, v)
    return write


def unsafe_rows(schema: StructType, rows: Sequence[Sequence], opts: Opts, ptypes=(), pvalues=()):
    """the UnsafeRows tfr_batch_rows (with partition values: tfr_batch_rows_with_partition) gives for read rows, which are
    also tfr_encode_rows' input -> (uint8 rows, int64 offsets)"""
    return PR.joined_rows(schema, rows, list(ptypes), list(pvalues), write_field(opts))


# ---- seeded composed schemas and rows ----
LEAVES = {
    "long": (LongType(), lambda r: int(r.integers(-2**40, 2**40))),
    "int": (IntegerType(), lambda r: int(r.integers(-2**31, 2**31))),
    "float": (FloatType(), lambda r: float(np.float32(r.standard_normal()))),
    "double": (DoubleType(), lambda r: float(np.float32(r.standard_normal() * 1e3))),    # (written as a FloatList)
    "string": (StringType(), lambda r: "s" * int(r.integers(0, 4)) + "é" * int(r.integers(0, 2))),
    "binary": (BinaryType(), lambda r: bytes(r.integers(0, 256, int(r.integers(0, 5)), dtype=np.uint8))),
}
# INT64 TYPES leaves as their columns hold them, inside what datetime.date / datetime.datetime hold; EDGES where a type allows
_RANGE = {A.TFR_T_INT8: (-128, 128), A.TFR_T_INT16: (-32768, 32768), A.TFR_T_DATE: (-719162, 2932897),
          A.TFR_T_TIMESTAMP: (-62135596800 * 10**6, 253402300799 * 10**6)}


def int64_gen(t: int):
    if t == A.TFR_T_BOOL:
        return lambda r: int(r.integers(0, 2))
    lo, hi = _RANGE[t]
    return lambda r: int(r.integers(lo, hi))


def _nonzero(r):
    x = float(np.float32(r.standard_normal()))
    return x if x != 0.0 else 1.0


def vector_gen(r):
    if r.integers(0, 2):
        return DenseVector([_nonzero(r) if r.integers(0, 4) else 0.0 for _ in range(int(r.integers(0, 7)))])
    size = int(r.integers(1, 40))
    idx = sorted(set(int(x) for x in r.integers(0, size, int(r.integers(0, 5)))))
    return SparseVector(size, idx, [_nonzero(r) for _ in idx])


def field_kinds(ragged: bool, extended: bool) -> List[str]:
    """what a seeded field is drawn from: plain leaves at depth 0 and 1 (2: ragged), vectors, INT64 TYPES at depth 0, 1, 2"""
    kinds = [f"{leaf}:{d}" for leaf in LEAVES for d in ((0, 1, 2) if ragged else (0, 1))] + ["vector"]
    if extended:
        kinds += [f"{name}:{d}" for name in I.TYPES for d in ((0, 1, 2) if ragged else (0, 1))]
    return kinds


def make_field(name: str, kind: str, nullable: bool) -> StructField:
    if kind == "vector":
        return StructField(name, VectorUDT(), nullable)
    leaf, d = kind.split(":")
    dt = LEAVES[leaf][0] if leaf in LEAVES else I.TYPES[leaf][0]
    for _ in range(int(d)):
        dt = ArrayType(dt)
    return StructField(name, dt, nullable)


def value_gen(f, opts: Opts):
    """a generator of f's values (rng -> value) in the row conventions above"""
    if isinstance(f.dataType, VectorUDT):
        return vector_gen
    depth, dt = 0, f.dataType
    while isinstance(dt, ArrayType):
        depth, dt = depth + 1, dt.elementType
    t = _i64(f, opts)
    leaf = int64_gen(t) if t else next(g for (lt, g) in LEAVES.values() if lt == dt)
    if depth == 0:
        return leaf
    if depth == 1:
        return lambda r: [leaf(r) for _ in range(int(r.integers(0, 5)))]
    return lambda r: [[leaf(r) for _ in range(int(r.integers(0, 4)))] for _ in range(int(r.integers(0, 4)))]


def seeded_schema(seed: int, n: int, opts: Opts, kinds: Optional[List[str]] = None) -> StructType:
    """n fields drawn from field_kinds (interleaved, so the parts of sparse and ragged fields are not next to their owners)"""
    r = np.random.default_rng(seed)
    kinds = kinds or field_kinds(opts.ragged, opts.extended_types)
    return StructType([make_field(f"c{i}", kinds[int(r.integers(0, len(kinds)))], bool(r.integers(0, 4))) for i in range(n)])


def with_kinds(schema: StructType, seed: int, named_kinds) -> StructType:
    """the schema with a field of each (name, kind) inserted at a seeded place"""
    r = np.random.default_rng(seed + 2000)
    fields = list(schema.fields)
    for nm, kind in named_kinds:
        fields.insert(int(r.integers(0, len(fields) + 1)), make_field(nm, kind, True))
    return StructType(fields)


def with_extras(schema: StructType, seed: int, corrupt: bool) -> Tuple[StructType, Optional[int]]:
    """the schema with the two generated fields and (corrupt) a corrupt-record column at seeded positions -> (schema, its
    index)"""
    r = np.random.default_rng(seed + 1000)
    fields = list(schema.fields)
    extras = [StructField("_tmp_metadata_row_index", RowIndexType(), False),
              StructField("_tmp_metadata_record_offset", RecordOffsetType(), False)]
    if corrupt:
        extras.append(StructField("_corrupt_record", BinaryType(), True))
    for f in extras:
        fields.insert(int(r.integers(0, len(fields) + 1)), f)
    idx = next((i for i, f in enumerate(fields) if f.name == "_corrupt_record"), None)
    return StructType(fields), idx


def seeded_rows(schema: StructType, opts: Opts, n: int, seed: int) -> List[tuple]:
    """rows of the writer's schema; about one in five values of a nullable field null"""
    r = np.random.default_rng(seed)
    gens = [value_gen(f, opts) for f in schema]
    return [tuple(None if f.nullable and r.integers(0, 5) == 0 else g(r) for f, g in zip(schema, gens)) for _ in range(n)]


def read_rows(schema: StructType, data: bytes, opts: Opts) -> List[tuple]:
    """every record of a clean file read back (errors raise)"""
    out = []
    for e in RW.chain(data, 0, True)[0]:
        row, err = read(schema, data[e[1] + 12:e[2] - 4], opts)
        assert err is None, err
        out.append(row)
    return out


# ---- the count boundaries ----
def boundary_schema(target, opts):
    """a caller's schema of target - 30 fields that lowers to `target` fields: `pad`, 10 sparse vectors (2 parts each) and
    10 ragged fields (1 part each) interleaved with plain fields"""
    assert opts.vector_format == "sparse" and opts.ragged
    n = target - 30
    kinds = ["vector"] * 10 + ["long:2"] * 5 + ["string:2"] * 5 + [("long:0", "float:1", "string:0")[i % 3] for i in range(n - 21)]
    r = np.random.default_rng(target)
    kinds = [kinds[i] for i in r.permutation(len(kinds))]
    return StructType([StructField("pad", ArrayType(LongType()), True)] +
                      [make_field(f"c{i}", k, True) for i, k in enumerate(kinds)])


def narrowed_schema(n):
    """`id`, n narrowed fields (BooleanType .. DateType at depth 0, 1 and 2) and a timestamp after every fifth, which is not
    narrowed"""
    kinds = ["bool", "byte", "short", "date"]
    fields = [StructField("id", LongType(), False)]
    for i in range(n):
        fields.append(make_field(f"n{i}", f"{kinds[i % 4]}:{(0, 1, 0, 2)[(i // 4) % 4]}", True))
        if i % 5 == 4:
            fields.append(make_field(f"t{i}", f"timestamp:{i % 2}", True))
    return StructType(fields)
