"""GPU tests of the VectorUDT field (include/tfrgpu.h, VECTORS).
  Decode : every case of tests/cases.py and every golden vector, with its scalar and 1-D fields as VectorUDT, gives the
           columns, tfr_batch_info and tfr_batch_dropped of the same schema with those fields as ArrayType(DoubleType), in
           FAILFAST, DROPMALFORMED, PERMISSIVE and PERMISSIVE + resync, on the tile / general / pipelined paths, and on the
           large-record path; the UnsafeRows (tfr_batch_rows, _with_partition, _async) are the dense structs of
           tests/vector_rows.py.
  Encode : columns are byte-identical to ArrayType(DoubleType); rows (dense and sparse, seeded) give pyref's / the oracle's
           bytes of toArray as ArrayType(DoubleType); the pipelined submit stays pipelined on a steady stream and redoes a
           batch far from what it learned; every malformed-struct clause is TFR_E_INVALID_ARG at its row; a densified batch
           above the encoder's limits is TFR_E_BATCH_TOO_LARGE.
  Round trip through the C ABI and through io.DefaultSource."""
import numpy as np
import pytest

import partition_rows as PR
import vector_rows as V
from cases import all_cases
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_encode_rows import rows_of
from test_golden import INDEX, schema_of
import os

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

MODES = {"failfast": None, "drop": A.TFR_F_VERIFY_CRC | A.TFR_F_DROP_MALFORMED, "permissive": A.TFR_F_VERIFY_CRC | A.TFR_F_PERMISSIVE,
         "permissive_resync": A.TFR_F_VERIFY_CRC | A.TFR_F_PERMISSIVE | A.TFR_F_RESYNC}


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def _swap(schema, make):
    """every data field of depth <= 1 (generated fields aside) as make(field)"""
    out = []
    for f in schema:
        t, d = lower_type(f.dataType)
        out.append(StructField(f.name, make(), f.nullable) if d <= 1 and t < TFR_T_ROW_INDEX else f)
    return StructType(out)


def _inputs():
    for c in all_cases():
        yield c.name, c.schema, c.record_type, c.data(), c.is_final, c.flags
    for e in INDEX:
        with open(os.path.join(HERE, "golden", e["file"]), "rb") as fh:
            data = fh.read()
        yield "golden:" + e["name"], schema_of(e), e["record_type"], data, e["is_final"], e["flags"]


INPUTS = list(_inputs())


def _snapshot(batch):
    cols = batch.to_host()
    return (dict(batch.info), [(c.elem_type, c.depth, c.null_count, None if c.validity is None else c.validity.tobytes(),
                                [o.tobytes() for o in c.offsets], c.values.tobytes()) for c in cols], batch.dropped())


def _decode_all(native, sch, rt, data, is_final, flags, general, monkeypatch):
    """(sync decode, pipelined submit after it) on one decoder: their snapshots and the decoder's counters"""
    if general:
        monkeypatch.setenv("TFR_DISABLE_FAST", "1")
    dec = native.Decoder(sch, rt, flags=flags)
    monkeypatch.delenv("TFR_DISABLE_FAST", raising=False)
    try:
        b, _ = dec.decode(data, is_final=is_final)
        s1 = _snapshot(b)
        b.release()
        b = dec.submit(data, is_final=is_final)
        s2 = _snapshot(b)
        b.release()
        return s1, s2, dec.stats()
    finally:
        dec.close()


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("general", [False, True], ids=["tile", "general"])
def test_decode_equals_double_arrays(native, monkeypatch, mode, general):
    n_checked = n_general = 0
    for name, sch, rt, data, is_final, flags in INPUTS:
        f = MODES[mode] if MODES[mode] is not None else flags
        if rt == TFR_RT_BYTE_ARRAY and f & A.TFR_F_PERMISSIVE:
            continue
        sv = _swap(sch, VectorUDT)
        sd = _swap(sch, lambda: ArrayType(DoubleType()))
        try:
            want = _decode_all(native, sd, rt, data, is_final, f, general, monkeypatch)
        except native.TfrError as e:                     # (a schema the decoder refuses in this mode refuses the vectors too)
            with pytest.raises(native.TfrError) as e2:
                _decode_all(native, sv, rt, data, is_final, f, general, monkeypatch)
            assert e2.value.code == e.code, name
            continue
        got = _decode_all(native, sv, rt, data, is_final, f, general, monkeypatch)
        assert got[0] == want[0], f"{name} ({mode}): sync decode differs"
        assert got[1] == want[1], f"{name} ({mode}): pipelined decode differs"
        n_general += got[2]["general_path_batches"] >= 1
        n_checked += 1
    assert n_checked > 100
    assert (n_general > 100) if general else n_general < n_checked, n_general


# ---- UnsafeRows of decoded vectors ---------------------------------------------------------------------------------------

def _vec_rows(sch_v, cols, n):
    """expected rows of the vector schema from the ArrayType(DoubleType) decode's columns (exact bits)"""
    rows = rows_of(cols, n)
    return [tuple(DenseVector(np.array(v, dtype=np.float64)) if isinstance(f.dataType, VectorUDT) and v is not None else v
                  for f, v in zip(sch_v, r)) for r in rows]


def _joined(sch_v, rows, ptypes, pvalues):
    parts = []
    for row in rows:
        w = PR._Writer(len(sch_v) + len(ptypes))
        for i, (f, v) in enumerate(zip(sch_v, row)):
            t, depth = lower_type(f.dataType)
            if v is None or t == TFR_T_NULL:
                w.set_null(i)
            elif isinstance(f.dataType, VectorUDT):
                w.var(i, V.vector_struct(v))
            elif depth == 0 and t not in (TFR_T_STRING, TFR_T_BINARY):
                w.slot(i, PR.U._scalar_bits(t, v))
            else:
                w.var(i, PR.U._leaf_bytes(t, v) if depth == 0 else PR.U.unsafe_array(t, depth, v))
        for j, (t, v) in enumerate(zip(ptypes, pvalues)):
            PR._write_partition(w, len(sch_v) + j, t, v)
        parts.append(w.row())
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(p) for p in parts])
    return np.frombuffer(b"".join(parts), dtype=np.uint8), offs


def _embedding_data(n, seed, max_len=48, big=0):
    """Examples: id, a FloatList `emb` (absent in every 7th row; `big` floats each when big > 0), a string"""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(n):
        feats = {"id": pyref.int64_feature(int(rng.integers(-2**40, 2**40))),
                 "s": pyref.bytes_feature(b"x" * int(rng.integers(0, 9)))}
        if r % 7 != 3:
            k = big if big else int(rng.integers(0, max_len))
            feats["emb"] = pyref.float_feature(*rng.standard_normal(k).astype(np.float32).tolist())
        out.append(pyref.frame(pyref.example(feats).SerializeToString()))
    return b"".join(out)


SCH_V = StructType([StructField("id", LongType()), StructField("emb", VectorUDT()), StructField("s", StringType()),
                    StructField("row", RowIndexType(), False)])
SCH_D = V.as_double_schema(SCH_V)


def _rows_ok(native, batch_d, batch_v, partition=None, ptv=None):
    cols = batch_d.to_host()
    n = batch_d.n_rows
    rows = _vec_rows(SCH_V, cols, n)
    if partition is None:
        wr, wo = V.unsafe_rows(SCH_V, rows)
        wo = wo.astype(np.int64)
        gr, go = batch_v.unsafe_rows(to_host=True)
    else:
        wr, wo = _joined(SCH_V, rows, *ptv)
        gr, go = batch_v.unsafe_rows(to_host=True, partition=partition)
    assert np.array_equal(go, wo) and np.array_equal(gr, wr)


@pytest.mark.parametrize("big", [0, 4096], ids=["tile", "large_record"])
def test_rows_of_decoded_vectors(native, big):
    data = _embedding_data(300 if big else 3000, seed=5 + big, big=big)
    dd, dv = native.Decoder(SCH_D), native.Decoder(SCH_V)
    try:
        bd, _ = dd.decode(data)
        bv, _ = dv.decode(data)
        assert _snapshot(bd) == _snapshot(bv)
        _rows_ok(native, bd, bv)
        if big:
            assert dv.stats()["large_record_batches"] >= 1, dv.stats()
        ptypes, pvalues = ["string", "int", ("decimal", 38, 6)], ["part=7", -3, 12345678901234567890]
        bv2, _ = dv.decode(data)
        _rows_ok(native, bd, bv2, (PR.partition_row(ptypes, pvalues), PR.var_flags(ptypes)), (ptypes, pvalues))
        for b in (bd, bv, bv2):
            b.release()
        # the asynchronous rows: learned on the first batch, enqueued at submit on the next ones
        for k in range(3):
            b1 = dd.submit(data)
            b2 = dv.submit(data)
            b2.unsafe_rows_async(to_host=True)
            _rows_ok(native, b1, b2)
            b1.release()
            b2.release()
        st = dv.stats()
        assert st["rows_async"] >= 1 and st["speculative_submits"] >= 1, st
    finally:
        dd.close()
        dv.close()


def test_rows_of_corrupt_and_generated_fields(native):
    data = bytearray(_embedding_data(500, seed=9))
    offs = []
    p = 0
    while p < len(data):
        offs.append(p)
        p += 16 + int.from_bytes(data[p:p + 8], "little")
    for r in (3, 100, 411):                                   # payload CRC flips: corrupt rows
        data[offs[r] + 13] ^= 0x40
    for flags in (A.TFR_F_VERIFY_CRC | A.TFR_F_PERMISSIVE, A.TFR_F_VERIFY_CRC | A.TFR_F_DROP_MALFORMED):
        dd, dv = native.Decoder(SCH_D, flags=flags), native.Decoder(SCH_V, flags=flags)
        try:
            bd, _ = dd.decode(bytes(data), first_entry=10, first_offset=1000)
            bv, _ = dv.decode(bytes(data), first_entry=10, first_offset=1000)
            assert _snapshot(bd) == _snapshot(bv) and len(bv.dropped()) == 3
            _rows_ok(native, bd, bv)
            bd.release()
            bv.release()
        finally:
            dd.close()
            dv.close()


# ---- encode ---------------------------------------------------------------------------------------------------------------

def _columns(sch_v, rows):
    """the ArrayType(DoubleType) columns of vector rows, built with numpy (vectors of 2^18 values)"""
    cols = []
    for i, f in enumerate(sch_v):
        if not isinstance(f.dataType, VectorUDT):
            cols.append(A.columns_from_rows(StructType([f]), [(r[i],) for r in rows])[0])
            continue
        n = len(rows)
        valid = np.zeros((n + 7) // 8, np.uint8)
        parts, offs = [], [0]
        for r, row in enumerate(rows):
            v = row[i]
            if v is not None:
                valid[r >> 3] |= 1 << (r & 7)
                parts.append(v.toArray())
            offs.append(offs[-1] + (0 if v is None else v.size))
        vals = np.concatenate(parts) if parts else np.zeros(0)
        cols.append(A.HostColumn(TFR_T_FLOAT64, 1, n, valid, [np.array(offs, np.int32)], vals))
    return cols


def _want(oracle, sch_v, rows, rt=0):
    sd = V.as_double_schema(sch_v)
    data, rc, _ = oracle.encode(_columns(sch_v, rows), sd, rt)
    assert rc == 0
    return data


def _rand_rows(rng, n, dense_max=4096, sparse_max=1 << 18, nnz_max=200, nullable=True):
    rows = []
    for r in range(n):
        k = rng.integers(0, 4)
        if k == 0 and nullable:
            v = None
        elif k == 1:
            v = DenseVector(rng.standard_normal(int(rng.integers(0, dense_max + 1))))
        else:
            size = int(rng.integers(0, sparse_max + 1))
            nnz = min(size, int(rng.integers(0, nnz_max + 1)))
            idx = np.sort(rng.choice(size, nnz, replace=False)) if nnz else np.zeros(0, np.int32)
            v = SparseVector(size, idx, rng.standard_normal(nnz) * 1e3)
        rows.append((int(rng.integers(-2**31, 2**31)), v, float(rng.standard_normal())))
    return rows


SCH_E = StructType([StructField("id", LongType()), StructField("v", VectorUDT()), StructField("label", DoubleType())])


def test_encode_columns_identical(native, oracle):
    rows = _rand_rows(np.random.default_rng(1), 200, sparse_max=5000)
    cols = A.columns_from_rows(SCH_E, rows)
    ev, ed = native.Encoder(SCH_E), native.Encoder(V.as_double_schema(SCH_E))
    try:
        got = ev.encode(cols)
        assert got == ed.encode(cols) == _want(oracle, SCH_E, rows)
    finally:
        ev.close()
        ed.close()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_encode_rows_dense_and_sparse(native, oracle, seed):
    rng = np.random.default_rng(100 + seed)
    rows = _rand_rows(rng, 64 if seed < 2 else 400, sparse_max=(1 << 18) if seed < 2 else 300)
    rows[0] = (1, SparseVector(0, [], []), 0.5)
    rows[1] = (2, DenseVector([]), 0.25)
    rows[2] = (3, SparseVector(1 << 18, [0, (1 << 18) - 1], [1.0, -2.0]), 0.0)
    want = _want(oracle, SCH_E, rows)
    # pyref's DoubleType rule on a sample (the C oracle encodes the same columns)
    sd = V.as_double_schema(SCH_E)
    for r in (0, 1, 2, 5):
        assert pyref.frame(pyref.serialize_example_bytes(sd, V.as_double_rows(SCH_E, [rows[r]])[0])) in want
    data, offs = V.unsafe_rows(SCH_E, rows)
    enc = native.Encoder(SCH_E)
    try:
        enc.encode_rows(data, offs)
        assert enc.result_host() == want
        s = enc.submit_rows(data, offs)
        assert s.result_host() == want
        s.release()
    finally:
        enc.close()
    # and read back: the dense struct of toArray through float
    dec = native.Decoder(SCH_E)
    try:
        b, _ = dec.decode(want)
        got_rows, got_offs = b.unsafe_rows()
        exp = [(i, None if v is None else DenseVector(v.toArray().astype(np.float32).astype(np.float64)), lab) for i, v, lab in rows]
        # the label is DoubleType: written through toFloat, read back widened
        exp = [(i, v, float(np.float32(lab))) for i, v, lab in exp]
        wr, wo = V.unsafe_rows(SCH_E, exp)
        assert np.array_equal(got_offs, wo.astype(np.int64)) and np.array_equal(got_rows, wr)
        b.release()
    finally:
        dec.close()


def test_encode_rows_struct_read_as_spark_does(native, oracle):
    """type and size slots read whatever their null bits; the element null bits of indices and values ignored"""
    vals = V.double_array([1.0, 2.0])
    vals_null_elem = bytearray(vals)
    vals_null_elem[8] |= 0b10                                         # element 1 null: its slot's bits are copied
    rows = [(1, V.RawVector(V.struct_bytes(1, None, None, vals, type_null=True)), 0.0),
            (2, V.RawVector(V.struct_bytes(1, 77, V.int_array([5]), vals)), 0.0),       # dense: size and indices ignored
            (3, V.RawVector(V.struct_bytes(1, None, None, bytes(vals_null_elem))), 0.0),
            (4, V.RawVector(V.struct_bytes(0, 3, V.int_array([2]), V.double_array([9.0]))), 0.0)]
    ref = [(1, DenseVector([1.0, 2.0]), 0.0), (2, DenseVector([1.0, 2.0]), 0.0), (3, DenseVector([1.0, 2.0]), 0.0),
           (4, SparseVector(3, [2], [9.0]), 0.0)]
    enc = native.Encoder(SCH_E)
    try:
        enc.encode_rows(*V.unsafe_rows(SCH_E, rows))
        assert enc.result_host() == _want(oracle, SCH_E, ref)
    finally:
        enc.close()


def _bad_structs():
    good = V.vector_struct(SparseVector(4, [1], [1.0]))
    far = bytearray(V.vector_struct(DenseVector([1.0])))
    far[32:40] = ((4000 << 32) | 16).to_bytes(8, "little")         # values slot outside the struct
    bad_arr = (1000).to_bytes(8, "little") + b"\0" * 16             # numElements past the array's bytes
    return {
        "slot_outside_row": V.RawVector(good, size=len(good) + 4096),
        "slot_misaligned": V.RawVector(good, offset_delta=4),
        "shorter_than_40": V.RawVector(good[:32], size=32),
        "type_2": V.RawVector(V.struct_bytes(2, None, None, V.double_array([1.0]))),
        "type_minus_1": V.RawVector(V.struct_bytes(0xFF, None, None, V.double_array([1.0]))),
        "null_values_dense": V.RawVector(V.struct_bytes(1, None, None, None)),
        "null_values_sparse": V.RawVector(V.struct_bytes(0, 4, V.int_array([1]), None)),
        "null_indices_sparse": V.RawVector(V.struct_bytes(0, 4, None, V.double_array([1.0]))),
        "values_outside_struct": V.RawVector(bytes(far)),
        "malformed_values_array": V.RawVector(V.struct_bytes(1, None, None, bad_arr)),
        "malformed_indices_array": V.RawVector(V.struct_bytes(0, 4, bad_arr, V.double_array([1.0]))),
        "size_negative": V.RawVector(V.struct_bytes(0, -1, V.int_array([]), V.double_array([]))),
        "lengths_differ": V.RawVector(V.struct_bytes(0, 4, V.int_array([0, 1]), V.double_array([1.0]))),
        "index_at_size": V.RawVector(V.struct_bytes(0, 4, V.int_array([4]), V.double_array([1.0]))),
        "index_negative": V.RawVector(V.struct_bytes(0, 4, V.int_array([-1]), V.double_array([1.0]))),
        "index_decreasing": V.RawVector(V.struct_bytes(0, 4, V.int_array([2, 1]), V.double_array([1.0, 2.0]))),
        "index_repeated": V.RawVector(V.struct_bytes(0, 4, V.int_array([1, 1]), V.double_array([1.0, 2.0]))),
    }


@pytest.mark.parametrize("clause", list(_bad_structs()))
def test_encode_rows_malformed_struct(native, clause):
    bad = _bad_structs()[clause]
    rows = [(r, DenseVector([float(r)]), 0.0) for r in range(6)]
    rows[4] = (4, bad, 0.0)
    data, offs = V.unsafe_rows(SCH_E, rows)
    enc = native.Encoder(SCH_E)
    try:
        with pytest.raises(native.TfrError) as e:
            enc.encode_rows(data, offs)
        assert e.value.code == A.TFR_E_INVALID_ARG and e.value.row == 4, (clause, e.value.code, e.value.row)
        s = enc.submit_rows(data, offs)
        with pytest.raises(native.TfrError) as e:
            s.wait()
        assert e.value.code == A.TFR_E_INVALID_ARG and e.value.row == 4
        s.release()
    finally:
        enc.close()


def test_encode_rows_null_and_precedence(native):
    sch = StructType([StructField("id", LongType()), StructField("v", VectorUDT(), False)])
    bad = _bad_structs()["type_2"]
    enc = native.Encoder(sch)
    try:
        for rows, code, row in [([(0, DenseVector([1.0])), (1, None), (2, bad)], A.TFR_E_NULL_IN_NONNULL, 1),
                                ([(0, DenseVector([1.0])), (1, bad), (2, None)], A.TFR_E_INVALID_ARG, 1),
                                ([(0, None), (1, bad)], A.TFR_E_NULL_IN_NONNULL, 0)]:
            with pytest.raises(native.TfrError) as e:
                enc.encode_rows(*V.unsafe_rows(sch, rows))
            assert (e.value.code, e.value.row) == (code, row)
    finally:
        enc.close()


def test_encode_rows_densify_too_large(native):
    rows = [(1, SparseVector(600_000_000, [5], [1.0]), 0.0)]
    data, offs = V.unsafe_rows(SCH_E, rows)
    enc = native.Encoder(SCH_E)
    try:
        with pytest.raises(native.TfrError) as e:
            enc.encode_rows(data, offs)
        assert e.value.code == A.TFR_E_BATCH_TOO_LARGE
        small = V.unsafe_rows(SCH_E, [(1, DenseVector([1.0]), 0.0)] * 100)
        for _ in range(2):                                          # learned, then pipelined
            enc.submit_rows(*small).release()
        s = enc.submit_rows(data, offs)
        with pytest.raises(native.TfrError) as e:
            s.wait()
        assert e.value.code == A.TFR_E_BATCH_TOO_LARGE
        s.release()
    finally:
        enc.close()


def _steady(rng, n):
    rows = []
    for r in range(n):
        idx = np.sort(rng.choice(4096, 64, replace=False))
        rows.append((r, SparseVector(4096, idx, rng.standard_normal(64)), 1.0))
    return rows


def test_encode_rows_submit_pipelined(native, oracle):
    rng = np.random.default_rng(7)
    enc = native.Encoder(SCH_E)
    try:
        batches = [_steady(rng, 500) for _ in range(8)]
        inflight = []                  # two in flight, each released before its lane is reused (a held result keeps the lane's buffers)
        for b in batches + [None, None]:
            if b is not None:
                inflight.append((enc.submit_rows(*V.unsafe_rows(SCH_E, b)), b))
            if len(inflight) > 2 or (b is None and inflight):
                s, w = inflight.pop(0)
                assert s.result_host() == _want(oracle, SCH_E, w)
                s.release()
        st = enc.stats()
        assert st["speculative_submits"] == 7 and st["speculative_redone"] == 0, st
        # far sparser (2^16-long vectors from as many bytes) and far denser (dense 64-value vectors) than what was learned
        sparse = [(r, SparseVector(1 << 16, np.sort(rng.choice(1 << 16, 64, replace=False)), rng.standard_normal(64)), 1.0) for r in range(100)]
        dense = [(r, DenseVector(rng.standard_normal(64)), 1.0) for r in range(500)]
        for b in (sparse, dense, batches[0]):
            s = enc.submit_rows(*V.unsafe_rows(SCH_E, b))
            assert s.result_host() == _want(oracle, SCH_E, b)
            s.release()
        st2 = enc.stats()
        assert st2["speculative_redone"] >= 1, st2
        # learned again: a steady stream of the sparser rows stays pipelined
        for _ in range(3):
            s = enc.submit_rows(*V.unsafe_rows(SCH_E, sparse))
            assert s.result_host() == _want(oracle, SCH_E, sparse)
            s.release()
        st3 = enc.stats()
        assert st3["speculative_redone"] <= st2["speculative_redone"] + 1, (st2, st3)
    finally:
        enc.close()


def test_round_trip_io(native, tmp_path):
    from spark_tfrecord_b200 import io as tio
    rng = np.random.default_rng(3)
    rows = _rand_rows(rng, 40, dense_max=50, sparse_max=300, nnz_max=20)
    tio.DefaultSource().save(str(tmp_path / "out"), SCH_E, rows)
    got = tio.DefaultSource().load(str(tmp_path / "out"), SCH_E)
    assert len(got) == len(rows)
    for (i, v, lab), (gi, gv, gl) in zip(rows, got):
        assert gi == i and gl == float(np.float32(lab))
        if v is None:
            assert gv is None
        else:
            assert isinstance(gv, DenseVector) and np.array_equal(gv.toArray(), v.toArray().astype(np.float32).astype(np.float64))
