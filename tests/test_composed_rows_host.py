"""CPU tests of tests/composed_rows.py: with one lowering on it gives what that lowering's own module gives, its writes read
back, and its lowered order and field counts are the library's."""
import numpy as np
import pytest

import composed_rows as CR
import int64_types as I
import ragged_rows as RR
import ragged_splits_rows as RS
import sparse_vector_rows as SP
import vector_rows as V
from oracle import pyref, unsaferow
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import sqltypes
from spark_tfrecord_b200.sqltypes import *  # noqa

SEEDS = range(12)


def _schema_of(kinds, nullable=True):
    return StructType([CR.make_field(f"c{i}", k, nullable) for i, k in enumerate(kinds)])


def _canon_rows(rows):
    return [CR.canon(list(r)) for r in rows]


# ---- one option on: exactly the per-feature module ----
@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("splits", [False, True])
def test_ragged_alone_is_the_ragged_module(seed, splits):
    M = RS if splits else RR
    opts = CR.Opts(ragged=True, row_splits=splits)
    sch = CR.seeded_schema(seed, 6, opts, [f"{leaf}:{d}" for leaf in CR.LEAVES for d in (0, 1, 2)])
    rows = CR.seeded_rows(sch, opts, 40, seed)
    assert CR.lowered_schema(sch, opts).fields == M.lowered_schema(sch).fields
    assert [CR.lower_row(sch, r, opts) for r in rows] == [M.lower_row(sch, r) for r in rows]
    data = CR.encode(sch, rows, opts)
    assert data == M.encode(sch, rows)
    for e in pyref_frames(data):
        assert CR.read(sch, e, opts) == M.read(sch, e)


def pyref_frames(data):
    import resync_walk as RW
    return [data[e[1] + 12:e[2] - 4] for e in RW.chain(data, 0, True)[0]]


@pytest.mark.parametrize("seed", SEEDS)
def test_sparse_alone_is_the_sparse_module(seed):
    opts = CR.Opts(vector_format="sparse")
    sch = CR.seeded_schema(seed, 7, opts, ["vector", "long:0", "float:1", "string:0"])
    rows = CR.seeded_rows(sch, opts, 30, seed)
    assert CR.lowered_schema(sch, opts).fields == sqltypes.lowered_schema(sch, "sparse").fields == SP.twin_schema(sch).fields
    assert [CR.lower_row(sch, r, opts) for r in rows] == SP.twin_rows(sch, rows)
    got = CR.unsafe_rows(sch, [CR.read(sch, p, opts)[0] for p in pyref_frames(CR.encode(sch, rows, opts))], opts)
    want = SP.unsafe_rows(sch, [tuple(SP.SparseParts(*CR._sparse_of(v)) if SP.is_vector(f) and v is not None else v
                                      for f, v in zip(sch, r)) for r in rows])
    assert got[0].tobytes() == want[0].tobytes() and list(got[1]) == list(want[1])


@pytest.mark.parametrize("seed", SEEDS)
def test_dense_alone_is_the_vector_module(seed):
    opts = CR.Opts()
    sch = CR.seeded_schema(seed, 6, opts, ["vector", "double:1", "int:0", "binary:0"])
    rows = CR.seeded_rows(sch, opts, 30, seed)
    assert CR.lowered_schema(sch, opts).fields == V.as_double_schema(sch).fields
    assert [CR.lower_row(sch, r, opts) for r in rows] == V.as_double_rows(sch, rows)
    got = CR.unsafe_rows(sch, rows, opts)
    want = V.unsafe_rows(sch, rows)
    assert got[0].tobytes() == want[0].tobytes() and list(got[1]) == list(want[1])


@pytest.mark.parametrize("seed", SEEDS)
def test_extended_alone_is_the_int64_module(seed):
    opts = CR.Opts(extended_types=True)
    sch = CR.seeded_schema(seed, 8, opts, [f"{n}:{d}" for n in I.TYPES for d in (0, 1)] + ["long:0", "float:0"])
    rows = CR.seeded_rows(sch, opts, 30, seed)
    assert CR.lowered_schema(sch, opts).fields == I.long_schema(sch).fields
    assert [CR.lower_row(sch, r, opts) for r in rows] == I.long_rows(sch, rows)
    got = CR.unsafe_rows(sch, rows, opts)
    want = b"".join(I.unsafe_row(sch, r) for r in rows)
    assert got[0].tobytes() == want
    # a read narrows: every EDGES value of a LongType feature
    for f_i, f in enumerate(sch):
        t = I.leaf_id(f.dataType)
        if not t or isinstance(f.dataType, ArrayType):
            continue
        for x in I.EDGES:
            row = list(I.long_rows(sch, [rows[0]])[0])
            row[f_i] = x
            got_row, err = CR.read(sch, pyref.serialize_example_bytes(I.long_schema(sch), row), opts)
            assert err is None and got_row[f_i] == int(I.narrow(t, np.array([x]))[0])


def test_partition_join_is_the_partition_module():
    import partition_rows as PR
    sch = StructType([StructField("a", LongType()), StructField("s", StringType()), StructField("x", ArrayType(FloatType()))])
    rows = [(1, "x", [1.5]), (None, "", None), (-3, None, [])]
    pt, pv = ["string", "int", ("decimal", 38, 6)], ["p", 4, 123]
    got = CR.unsafe_rows(sch, rows, CR.Opts(), pt, pv)
    want = PR.joined_rows(sch, rows, pt, pv)
    assert got[0].tobytes() == want[0].tobytes() and list(got[1]) == list(want[1])
    assert CR.unsafe_rows(sch, rows, CR.Opts())[0].tobytes() == unsaferow.unsafe_rows(sch, rows)[0].tobytes()


# ---- everything on: writes read back ----
OPTS = [CR.Opts(v, True, s, True) for v in ("dense", "sparse") for s in (False, True)]


@pytest.mark.parametrize("seed", SEEDS)
def test_composed_round_trip(seed):
    opts = OPTS[seed % len(OPTS)]
    sch = CR.seeded_schema(seed, 24, opts)
    rows = CR.seeded_rows(sch, opts, 25, seed)
    data = CR.encode(sch, rows, opts)
    back = CR.read_rows(sch, data, opts)
    assert _canon_rows(back) == _canon_rows(rows)
    # through the decoder's schema too: the generated fields and the corrupt-record column are no feature's
    dsch, corrupt = CR.with_extras(sch, seed, True)
    dopts = CR.Opts(opts.vector_format, True, opts.row_splits, True, corrupt)
    exp = CR.Expect(dsch, dopts, data, "PERMISSIVE")
    assert exp.error is None and not exp.dropped and len(exp.rows) == len(rows)
    extra = [i for i, f in enumerate(dsch) if f.name.startswith("_")]
    for r, (got, want) in enumerate(zip(exp.rows, rows)):
        assert CR.canon([v for i, v in enumerate(got) if i not in extra]) == CR.canon(list(want))
        assert got[corrupt] is None
    offs = [0] + list(np.cumsum([16 + len(p) for p in pyref_frames(data)]))[:-1]
    ri = dsch.names.index("_tmp_metadata_row_index")
    ro = dsch.names.index("_tmp_metadata_record_offset")
    assert [r[ri] for r in exp.rows] == list(range(len(rows))) and [r[ro] for r in exp.rows] == offs


def test_owner_of_every_part():
    """a part's error reports its vector or ragged field, with the parts of both interleaved with other fields"""
    opts = CR.Opts("sparse", True, False, True)
    sch = _schema_of(["long:0", "long:2", "vector", "int:1", "vector", "short:2", "float:0"])
    low = CR.lowered_schema(sch, opts)
    assert low.names == ["c0", "c1_values", "c2_values", "c3", "c4_values", "c5_values", "c6", "c2_indices", "c2_size",
                         "c4_indices", "c4_size", "c1_row_lengths", "c5_row_lengths"]
    assert [CR.owner(sch, opts, f) for f in range(len(low))] == [0, 1, 2, 3, 4, 5, 6, 2, 2, 4, 4, 1, 5]
    feats = {"c0": pyref.int64_feature(1), "c6": pyref.float_feature(1.0)}
    for bad, field in (("c2_indices", 2), ("c4_size", 4), ("c1_row_lengths", 1), ("c5_row_lengths", 5)):
        p = pyref.example({**feats, bad: pyref.bytes_feature(b"x")}).SerializeToString()
        assert CR.read(sch, p, opts) == (None, (A.TFR_E_KIND_MISMATCH, field))
    # two failing parts: the one earlier in the lowered order (the sparse part) is reported
    p = pyref.example({**feats, "c5_row_lengths": pyref.float_feature(1.0), "c4_indices": pyref.float_feature(1.0)})
    assert CR.read(sch, p.SerializeToString(), opts) == (None, (A.TFR_E_KIND_MISMATCH, 4))
    # a mismatch of ragged parts is checked after every part parsed
    p = pyref.example({**feats, "c1_values": pyref.int64_feature(1, 2), "c1_row_lengths": pyref.int64_feature(3)})
    assert CR.read(sch, p.SerializeToString(), opts) == (None, (A.TFR_E_BAD_NESTING, 1))


# ---- the library's counts ----
def _num_cols(sch, opts):
    from spark_tfrecord_b200 import _native
    s = _native.Schema(sch, 0, **opts.native())
    try:
        return _native.lib().tfr_schema_num_fields(s.h)
    finally:
        s.close()


@pytest.mark.parametrize("seed", SEEDS)
def test_lowered_counts(seed):
    opts = OPTS[seed % len(OPTS)]
    sch = CR.seeded_schema(seed, 40, opts)
    n_sp = sum(isinstance(f.dataType, VectorUDT) for f in sch) if opts.vector_format == "sparse" else 0
    n_rg = len(RR.ragged_fields(sch))
    assert CR.n_lowered(sch, opts) == len(CR.lowered_schema(sch, opts)) == len(sch) + 2 * n_sp + n_rg
    assert _num_cols(sch, opts) == len(sch) + 2 * n_sp                    # ragged parts are not columns
    assert CR.n_narrowed(sch, opts) == sum(1 for f in sch if I.leaf_id(f.dataType) not in (0, A.TFR_T_TIMESTAMP))


@pytest.mark.parametrize("target", [127, 128, 129])
def test_boundary_schemas_lower_to_their_count(target):
    for opts in [o for o in OPTS if o.vector_format == "sparse"]:
        sch = CR.boundary_schema(target, opts)
        assert CR.n_lowered(sch, opts) == target
        assert any(isinstance(f.dataType, VectorUDT) for f in sch) and RR.ragged_fields(sch)
        assert _num_cols(sch, opts) == target - len(RR.ragged_fields(sch))


@pytest.mark.parametrize("n", [64, 65, 128, 129])
def test_narrowed_boundary_schemas(n):
    sch = CR.narrowed_schema(n)
    opts = CR.Opts(ragged=True, extended_types=True)
    assert CR.n_narrowed(sch, opts) == n
    assert any(I.leaf_id(f.dataType) == A.TFR_T_TIMESTAMP for f in sch)


# ---- one option on, over the corpora the per-feature suites decode ----
@pytest.mark.parametrize("splits", [False, True])
def test_ragged_corpora(splits):
    """the row corpora and the corpus of records with bad parts of the ragged GPU suites: the same bytes and reads"""
    import test_gpu_ragged as G
    import test_gpu_ragged_splits as GS
    M, G = (RS, GS) if splits else (RR, G)
    opts = CR.Opts(ragged=True, row_splits=splits)
    for leaf in G.LEAVES:
        for nullable in (True, False):
            sch, rows = G._schema(leaf, nullable), G._rows(leaf, nullable, n=60)
            data = CR.encode(sch, rows, opts)
            assert data == M.encode(sch, rows)
            for p in pyref_frames(data):
                assert CR.read(sch, p, opts) == M.read(sch, p)
    sch = G._schema("long", True)
    bad = G._bad_records()
    assert any(M.read(sch, p)[1] is not None for p in bad)
    assert [CR.read(sch, p, opts) for p in bad] == [M.read(sch, p) for p in bad]


def test_int64_corpora():
    """the row corpora of the extendedTypes GPU suite: the LongType rows it writes, and the narrow rows it reads back"""
    import test_gpu_int64_types as G
    opts = CR.Opts(extended_types=True)
    for name in G.NAMES:
        for depth in (0, 1):
            for nullable in (True, False):
                sch, rows = G._schema(name, nullable, depth), G._rows(name, nullable, depth, n=60, seed=depth)
                assert [CR.lower_row(sch, r, opts) for r in rows] == I.long_rows(sch, rows)
                data = CR.encode(sch, rows, opts)
                assert data == G._pyref_bytes(sch, rows)
                assert CR.read_rows(sch, data, opts) == [tuple(r) for r in rows]
