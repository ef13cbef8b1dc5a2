"""GPU tests of the sparse-format VectorUDT field (include/tfrgpu.h, SPARSE VECTORS).  Every expectation comes from the lowered
twin schema -- the same fields, each sparse vector replaced by its three ordinary fields -- whose paths the rest of the suite
pins against the oracle.
  Decode : every case of tests/cases.py and every golden vector with a sparse vector added, and Examples whose parts are
           malformed, give the twin's columns, tfr_batch_info and tfr_batch_dropped (the field mapped to the vector), in
           FAILFAST, DROPMALFORMED, PERMISSIVE and PERMISSIVE + resync, on the tile / general / pipelined paths and on the
           large-record path; the UnsafeRows (tfr_batch_rows, _with_partition, _async) are tests/sparse_vector_rows.py's.
  Encode : seeded dense and sparse rows give the oracle's bytes of the twin rows; columns are byte-identical to the twin;
           decode -> columns -> tfr_encode reproduces the file; the pipelined submit stays pipelined and redoes an outlier;
           every malformed-struct clause fails at the row the dense format fails at; a batch over the densify limit encodes.
  Round trip through io.DefaultSource, and across the two formats."""
import os

import numpy as np
import pytest

import partition_rows as PR
import sparse_vector_rows as SV
import vector_rows as V
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_vector import INPUTS, MODES, _bad_structs, _snapshot, _steady

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def _decode_all(native, sch, rt, data, is_final, flags, general, monkeypatch, vf="dense"):
    """(sync decode, pipelined submit after it) on one decoder: their snapshots and the decoder's counters"""
    if general:
        monkeypatch.setenv("TFR_DISABLE_FAST", "1")
    dec = native.Decoder(sch, rt, flags=flags, vector_format=vf)
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


def _map_twin(snap, owner):
    """a twin decode's snapshot with its field indexes mapped as the sparse decode reports them (a part: its vector)"""
    info, cols, dropped = snap
    info = dict(info)
    info["error_field"] = owner.get(info["error_field"], info["error_field"])
    return info, cols, [tuple(owner.get(x, x) if k == 3 else x for k, x in enumerate(e)) for e in dropped]


def _owner(sch):
    nf = len(sch)
    sp = [i for i, f in enumerate(sch) if SV.is_vector(f)]
    return {nf + 2 * j + k: i for j, i in enumerate(sp) for k in (0, 1)}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("general", [False, True], ids=["tile", "general"])
def test_decode_cases_equal_twin(native, monkeypatch, mode, general):
    """every input with a sparse vector `sv` added (absent from the records: the parts are null) reads as its twin"""
    n_checked = 0
    for name, sch, rt, data, is_final, flags in INPUTS:
        f = MODES[mode] if MODES[mode] is not None else flags
        if rt == TFR_RT_BYTE_ARRAY and f & A.TFR_F_PERMISSIVE:
            continue
        ss = StructType(list(sch) + [StructField("sv", VectorUDT())])
        tw = SV.twin_schema(ss)
        try:
            want = _decode_all(native, tw, rt, data, is_final, f, general, monkeypatch)
        except native.TfrError as e:
            with pytest.raises(native.TfrError) as e2:
                _decode_all(native, ss, rt, data, is_final, f, general, monkeypatch, "sparse")
            assert e2.value.code == e.code, name
            continue
        got = _decode_all(native, ss, rt, data, is_final, f, general, monkeypatch, "sparse")
        own = _owner(ss) if rt != TFR_RT_BYTE_ARRAY else {}
        assert got[0] == _map_twin(want[0], own), f"{name} ({mode}): sync decode differs"
        assert got[1] == _map_twin(want[1], own), f"{name} ({mode}): pipelined decode differs"
        n_checked += 1
    assert n_checked > 100


def _parts_data(n, seed, big=0, bad=()):
    """Examples with the parts of sparse vectors `a` and `b`, an id and a string; rows in `bad` have a part of the wrong kind
    (a's size as a BytesList, b's indices as a FloatList, or a's values as an Int64List, in turn)"""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(n):
        feats = {"id": pyref.int64_feature(r), "s": pyref.bytes_feature(b"y" * (r % 5))}
        for v in ("a", "b"):
            if (r + (v == "b")) % 6 == 2:
                continue                                             # a null vector (its values absent)
            k = big if big else int(rng.integers(0, 40))
            if r % 11 != 4:
                feats[v + "_indices"] = pyref.int64_feature(*np.sort(rng.choice(1 << 18, k, replace=False)).tolist())
            feats[v + "_values"] = pyref.float_feature(*rng.standard_normal(k).astype(np.float32).tolist())
            if r % 13 != 5:
                feats[v + "_size"] = pyref.int64_feature(1 << 18)
        if r in bad:
            kind = bad.index(r) % 3
            if kind == 0:
                feats["a_size"] = pyref.bytes_feature(b"x")
            elif kind == 1:
                feats["b_indices"] = pyref.float_feature(1.0)
            else:
                feats["a_values"] = pyref.int64_feature(3)
        out.append(pyref.frame(pyref.example(feats).SerializeToString()))
    return b"".join(out)


SCH_P = StructType([StructField("id", LongType()), StructField("a", VectorUDT()), StructField("s", StringType()),
                    StructField("b", VectorUDT()), StructField("row", RowIndexType(), False)])


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("path", ["tile", "general", "large_record"])
def test_decode_malformed_parts_equal_twin(native, monkeypatch, mode, path):
    big = 3000 if path == "large_record" else 0
    data = _parts_data(200 if big else 2000, seed=3, big=big, bad=(17, 60, 61, 150, 151, 152))
    f = MODES[mode] if MODES[mode] is not None else A.TFR_F_VERIFY_CRC
    want = _decode_all(native, SV.twin_schema(SCH_P), 0, data, True, f, path == "general", monkeypatch)
    got = _decode_all(native, SCH_P, 0, data, True, f, path == "general", monkeypatch, "sparse")
    own = _owner(SCH_P)
    assert got[0] == _map_twin(want[0], own) and got[1] == _map_twin(want[1], own)
    if mode == "failfast":                                          # the first bad row: a's size, a part, reports a
        assert got[0][0]["error_row"] == 17 and got[0][0]["error_field"] == 1, got[0][0]
    else:
        assert {e[3] for e in got[0][2]} <= {1, 3} and len(got[0][2]) == 6, got[0][2]
    if big:                                                          # (a batch with a failing record is redone off that path)
        clean = _parts_data(200, seed=4, big=big)
        want = _decode_all(native, SV.twin_schema(SCH_P), 0, clean, True, f, False, monkeypatch)
        got = _decode_all(native, SCH_P, 0, clean, True, f, False, monkeypatch, "sparse")
        assert got[:2] == want[:2] and got[2]["large_record_batches"] >= 1, got[2]


# ---- UnsafeRows of decoded sparse vectors ----------------------------------------------------------------------------------

def _expected_rows(batch):
    cols = batch.to_host()
    return [SV.parts_of_columns(cols, SCH_P, r) for r in range(batch.n_rows)]


def _joined(rows, ptypes, pvalues):
    parts = []
    for row in rows:
        w = PR._Writer(len(SCH_P) + len(ptypes))
        one = SV.unsafe_rows(SCH_P, [row])[0].tobytes()
        nw = (len(SCH_P) + 63) // 64
        for i, (f, v) in enumerate(zip(SCH_P, row)):
            t, depth = lower_type(f.dataType)
            if v is None:
                w.set_null(i)
            elif isinstance(v, SV.SparseParts):
                w.var(i, SV.sparse_struct(v.size, v.indices, v.values))
            elif depth == 0 and t not in (TFR_T_STRING, TFR_T_BINARY):
                w.slot(i, int.from_bytes(one[8 * (nw + i):8 * (nw + i) + 8], "little"))
            else:
                w.var(i, PR.U._leaf_bytes(t, v))
        for j, (t, v) in enumerate(zip(ptypes, pvalues)):
            PR._write_partition(w, len(SCH_P) + j, t, v)
        parts.append(w.row())
    offs = np.zeros(len(parts) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(p) for p in parts])
    return np.frombuffer(b"".join(parts), dtype=np.uint8), offs


def _rows_ok(batch, partition=None, ptv=None):
    rows = _expected_rows(batch)
    if partition is None:
        wr, wo = SV.unsafe_rows(SCH_P, rows)
        gr, go = batch.unsafe_rows(to_host=True)
    else:
        wr, wo = _joined(rows, *ptv)
        gr, go = batch.unsafe_rows(to_host=True, partition=partition)
    assert np.array_equal(go, wo.astype(np.int64)) and np.array_equal(gr, wr)
    return rows


@pytest.mark.parametrize("big", [0, 3000], ids=["tile", "large_record"])
def test_rows_of_decoded_sparse_vectors(native, big):
    data = _parts_data(200 if big else 3000, seed=11 + big, big=big)
    dec = native.Decoder(SCH_P, vector_format="sparse")
    try:
        b, _ = dec.decode(data)
        rows = _rows_ok(b)
        # null sizes and null indices (their parts absent) with their vector present
        assert any(isinstance(r[1], SV.SparseParts) and r[1].size is None for r in rows)
        assert any(isinstance(r[1], SV.SparseParts) and r[1].indices is None for r in rows)
        b.release()
        ptypes, pvalues = ["string", "int", ("decimal", 38, 6)], ["part=7", -3, 12345678901234567890]
        b, _ = dec.decode(data)
        _rows_ok(b, (PR.partition_row(ptypes, pvalues), PR.var_flags(ptypes)), (ptypes, pvalues))
        b.release()
        # the asynchronous rows: learned on the first batch, enqueued at submit on the next ones; then a batch of far larger
        # rows than learned is redone by the rows call
        for k in range(3):
            b = dec.submit(data)
            b.unsafe_rows_async(to_host=True)
            _rows_ok(b)
            b.release()
        st = dec.stats()
        assert st["rows_async"] >= 1 and st["speculative_submits"] >= 1, st
        if not big:
            b = dec.submit(_parts_data(300, seed=12, big=600))
            b.unsafe_rows_async(to_host=True)
            _rows_ok(b)
            b.release()
    finally:
        dec.close()


# ---- encode ---------------------------------------------------------------------------------------------------------------

SCH_E = StructType([StructField("id", LongType()), StructField("v", VectorUDT()), StructField("label", DoubleType())])


def _rand_rows(rng, n, dense_max=4096, sparse_max=1 << 20, nnz_max=200):
    rows = []
    for r in range(n):
        k = rng.integers(0, 4)
        if k == 0:
            v = None
        elif k == 1:
            x = rng.standard_normal(int(rng.integers(0, dense_max + 1)))
            x[rng.random(len(x)) < 0.5] = 0.0                        # stored zeros, some -0.0, a NaN, a tiny double
            x[rng.random(len(x)) < 0.05] = -0.0
            if len(x) > 3:
                x[1], x[2] = np.nan, 1e-300
            v = DenseVector(x)
        else:
            size = int(rng.integers(0, sparse_max + 1))
            nnz = min(size, int(rng.integers(0, nnz_max + 1)))
            idx = np.sort(rng.choice(size, nnz, replace=False)) if nnz else np.zeros(0, np.int32)
            vals = rng.standard_normal(nnz) * 1e3
            vals[rng.random(nnz) < 0.2] = 0.0
            v = SparseVector(size, idx, vals)
        rows.append((int(rng.integers(-2**31, 2**31)), v, float(rng.standard_normal())))
    return rows


def _want(oracle, sch, rows, rt=0):
    tw = SV.twin_schema(sch)
    data, rc, _ = oracle.encode(A.columns_from_rows(tw, SV.twin_rows(sch, rows)), tw, rt)
    assert rc == 0
    return data


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_encode_rows_equal_twin(native, oracle, seed):
    rng = np.random.default_rng(200 + seed)
    rows = _rand_rows(rng, 64 if seed < 2 else 400, sparse_max=(1 << 20) if seed < 2 else 300)
    rows[0] = (1, SparseVector(0, [], []), 0.5)
    rows[1] = (2, DenseVector([]), 0.25)
    rows[2] = (3, SparseVector(1 << 20, [0, (1 << 20) - 1], [1.0, -2.0]), 0.0)
    rows[3] = (4, DenseVector(np.zeros(5)), 0.0)                   # the zero vector: empty values and indices, its size
    rows[4] = (5, DenseVector(rng.standard_normal(1 << 18)), 1.0)  # long dense vectors: the warp counts and compacts
    rows[5] = (6, DenseVector(np.where(rng.random(1 << 18) < 0.9, 0.0, 1.0)), 1.0)
    want = _want(oracle, SCH_E, rows)
    tw = SV.twin_schema(SCH_E)
    for r in (0, 1, 2, 3):                                        # pyref's rules on a sample (the C oracle encodes the same columns)
        assert pyref.frame(pyref.serialize_example_bytes(tw, SV.twin_rows(SCH_E, [rows[r]])[0])) in want
    data, offs = V.unsafe_rows(SCH_E, rows)
    enc = native.Encoder(SCH_E, vector_format="sparse")
    try:
        enc.encode_rows(data, offs)
        assert enc.result_host() == want
        s = enc.submit_rows(data, offs)
        assert s.result_host() == want
        s.release()
        # the columns path is the twin's, byte for byte
        cols = A.columns_from_rows(SCH_E, rows, vector_format="sparse")
        assert enc.encode(cols) == want
    finally:
        enc.close()
    # decode -> columns -> tfr_encode reproduces the file
    dec = native.Decoder(SCH_E, vector_format="sparse")
    enc = native.Encoder(SCH_E, vector_format="sparse")
    try:
        b, _ = dec.decode(want)
        assert enc.encode(b.to_host()) == want
        b.release()
    finally:
        dec.close()
        enc.close()


def test_encode_columns_equal_twin(native, oracle):
    rows = _rand_rows(np.random.default_rng(5), 300, sparse_max=5000)
    enc, et = native.Encoder(SCH_E, vector_format="sparse"), native.Encoder(SV.twin_schema(SCH_E))
    try:
        cols = A.columns_from_rows(SCH_E, rows, vector_format="sparse")
        assert enc.encode(cols) == et.encode(cols) == _want(oracle, SCH_E, rows)
    finally:
        enc.close()
        et.close()


def test_encode_rows_submit_pipelined(native, oracle):
    rng = np.random.default_rng(17)
    enc = native.Encoder(SCH_E, vector_format="sparse")
    try:
        batches = [_steady(rng, 500) for _ in range(8)]
        inflight = []
        for b in batches + [None, None]:
            if b is not None:
                inflight.append((enc.submit_rows(*V.unsafe_rows(SCH_E, b)), b))
            if len(inflight) > 2 or (b is None and inflight):
                s, w = inflight.pop(0)
                assert s.result_host() == _want(oracle, SCH_E, w)
                s.release()
        st = enc.stats()
        assert st["speculative_submits"] == 7 and st["speculative_redone"] == 0, st
        # an outlier far from what was learned (dense vectors, 64 non-zeros each of 4096 stored values), then the steady rows
        dense = [(r, DenseVector(np.where(rng.random(4096) < 64 / 4096, 1.0, 0.0)), 1.0) for r in range(200)]
        wide = [(r, DenseVector(rng.standard_normal(2048)), 1.0) for r in range(50)]
        for b in (dense, wide, batches[0]):
            s = enc.submit_rows(*V.unsafe_rows(SCH_E, b))
            assert s.result_host() == _want(oracle, SCH_E, b)
            s.release()
    finally:
        enc.close()


@pytest.mark.parametrize("clause", list(_bad_structs()))
def test_encode_rows_malformed_struct(native, clause):
    bad = _bad_structs()[clause]
    rows = [(r, DenseVector([float(r)]), 0.0) for r in range(6)]
    rows[4] = (4, bad, 0.0)
    data, offs = V.unsafe_rows(SCH_E, rows)
    for vf in ("dense", "sparse"):
        enc = native.Encoder(SCH_E, vector_format=vf)
        try:
            with pytest.raises(native.TfrError) as e:
                enc.encode_rows(data, offs)
            assert e.value.code == A.TFR_E_INVALID_ARG and e.value.row == 4, (vf, clause, e.value.code, e.value.row)
            s = enc.submit_rows(data, offs)
            with pytest.raises(native.TfrError) as e:
                s.wait()
            assert e.value.code == A.TFR_E_INVALID_ARG and e.value.row == 4
            s.release()
        finally:
            enc.close()


def test_encode_rows_null_in_non_nullable(native):
    sch = StructType([StructField("id", LongType()), StructField("v", VectorUDT(), False)])
    bad = _bad_structs()["type_2"]
    enc = native.Encoder(sch, vector_format="sparse")
    try:
        for rows, code, row in [([(0, DenseVector([1.0])), (1, None), (2, bad)], A.TFR_E_NULL_IN_NONNULL, 1),
                                ([(0, DenseVector([1.0])), (1, bad), (2, None)], A.TFR_E_INVALID_ARG, 1)]:
            with pytest.raises(native.TfrError) as e:
                enc.encode_rows(*V.unsafe_rows(sch, rows))
            assert (e.value.code, e.value.row) == (code, row)
    finally:
        enc.close()


def test_over_the_densify_limit_encodes_sparse(native, oracle):
    """4,096 HashingTF-like rows of size 2^18: 4 GiB dense, over the densify limit (TFR_E_BATCH_TOO_LARGE in dense format)"""
    rng = np.random.default_rng(23)
    rows = [(r, SparseVector(1 << 18, np.sort(rng.choice(1 << 18, 64, replace=False)), rng.standard_normal(64)), 1.0)
            for r in range(4096)]
    data, offs = V.unsafe_rows(SCH_E, rows)
    ed = native.Encoder(SCH_E)
    try:
        with pytest.raises(native.TfrError) as e:
            ed.encode_rows(data, offs)
        assert e.value.code == A.TFR_E_BATCH_TOO_LARGE
    finally:
        ed.close()
    enc = native.Encoder(SCH_E, vector_format="sparse")
    dec = native.Decoder(SCH_E, vector_format="sparse")
    try:
        enc.encode_rows(data, offs)
        out = enc.result_host()
        assert out == _want(oracle, SCH_E, rows)
        b, _ = dec.decode(out)
        got = SV.unsafe_rows(SCH_E, [SV.parts_of_columns(b.to_host(), SCH_E, r) for r in range(b.n_rows)])
        gr, go = b.unsafe_rows(to_host=True)
        assert np.array_equal(gr, got[0]) and np.array_equal(go, got[1].astype(np.int64))
        for r in (0, 4095):
            p = SV.parts_of_columns(b.to_host(), SCH_E, r)[1]
            assert p.size == 1 << 18 and list(p.indices) == rows[r][1].indices.tolist()
        b.release()
    finally:
        enc.close()
        dec.close()


def test_round_trip_io(native, tmp_path):
    from spark_tfrecord_b200 import io as tio
    rows = _rand_rows(np.random.default_rng(3), 60, dense_max=50, sparse_max=300, nnz_max=20)
    sparse = {"vectorFormat": "sparse"}
    tio.DefaultSource().save(str(tmp_path / "sp"), SCH_E, rows, sparse)
    got = tio.DefaultSource().load(str(tmp_path / "sp"), SCH_E, sparse)
    assert len(got) == len(rows)
    for (i, v, lab), (gi, gv, gl) in zip(rows, got):
        assert gi == i and gl == float(np.float32(lab))
        if v is None:
            assert gv is None
            continue
        s = v.toSparse()
        assert isinstance(gv, SparseVector) and gv.size == v.size and gv.indices.tolist() == s.indices.tolist()
        assert np.array_equal(gv.values, s.values.astype(np.float32).astype(np.float64), equal_nan=True)
    # the other format reads the vectors as null
    assert all(r[1] is None for r in tio.DefaultSource().load(str(tmp_path / "sp"), SCH_E))
    tio.DefaultSource().save(str(tmp_path / "dn"), SCH_E, rows)
    assert all(r[1] is None for r in tio.DefaultSource().load(str(tmp_path / "dn"), SCH_E, sparse))
    # a non-nullable vector read in the other format is an error
    strict = StructType([SCH_E[0], StructField("v", VectorUDT(), False), SCH_E[2]])
    with pytest.raises(native.TfrError) as e:
        list(tio.DefaultSource().load(str(tmp_path / "dn"), strict, sparse))
    assert e.value.code == A.TFR_E_NULL_IN_NONNULL
