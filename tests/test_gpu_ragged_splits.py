"""GPU tests of raggedPartition=rowSplits (include/tfrgpu.h, RAGGED, Row splits).  Every expectation comes from
tests/ragged_splits_rows.py: the writer's bytes are pyref's encoding of the lowered rows, and a read is the lowered parse raised
back into nested lists, or the record's error at the ragged field, in FAILFAST, DROPMALFORMED and PERMISSIVE (with and without
resync)."""
import numpy as np
import pytest

import ragged_rows as RR
import ragged_splits_rows as RS
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

pytestmark = pytest.mark.gpu

SPLITS = dict(ragged=True, row_splits=True)


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


LEAVES = {
    "long": (LongType(), lambda r: int(r.integers(-2**40, 2**40))),
    "int": (IntegerType(), lambda r: int(r.integers(-2**31, 2**31))),
    "float": (FloatType(), lambda r: float(np.float32(r.standard_normal()))),
    "double": (DoubleType(), lambda r: float(np.float32(r.standard_normal()))),
    "string": (StringType(), lambda r: "s" * int(r.integers(0, 5)) + "é"),
    "binary": (BinaryType(), lambda r: bytes(r.integers(0, 256, int(r.integers(0, 6)), dtype=np.uint8))),
    "decimal": (DecimalType(), lambda r: float(np.float32(r.integers(-10**6, 10**6) / 100.0))),
}
ROW_LEAVES = sorted(set(LEAVES) - {"decimal"})     # UnsafeRows: a DecimalType's layout depends on its declared precision


def _rows(leaf, nullable, n=300, seed=0):
    rng = np.random.default_rng(seed)
    gen = LEAVES[leaf][1]
    fixed = [[], [[]], [[], []], [[gen(rng) for _ in range(200)]]]
    rows = []
    for i in range(n):
        if i < len(fixed):
            x = fixed[i]
        elif nullable and i % 7 == 0:
            x = None
        elif i % 11 == 0:
            x = []
        else:
            x = [[gen(rng) for _ in range(int(rng.integers(0, 9)))] for _ in range(int(rng.integers(0, 33)))]
        rows.append((i, x, float(i)))
    return rows


def _schema(leaf, nullable):
    return StructType([StructField("id", LongType(), False),
                       StructField("x", ArrayType(ArrayType(LEAVES[leaf][0])), nullable),
                       StructField("w", FloatType(), True)])


def _norm(v):
    return v if v is None else [[float(np.float32(e)) if isinstance(e, float) else e for e in inner] for inner in v]


def test_exact_bytes_of_empty_and_null():
    sch = _schema("long", True)
    low = RS.lowered_schema(sch)
    assert RS.lower_row(sch, (0, [], 0.0))[3] == [0] and RS.lower_row(sch, (0, [[]], 0.0))[3] == [0, 0]
    assert RS.lower_row(sch, (0, None, 0.0))[1::2] == (None, None)
    assert low.fields[3].name == "x_row_splits"


@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("leaf", sorted(LEAVES))
def test_round_trip_and_bytes(native, leaf, nullable):
    sch = _schema(leaf, nullable)
    rows = _rows(leaf, nullable)
    enc = native.Encoder(sch, 0, **SPLITS)
    try:
        data = enc.encode(A.columns_from_rows(sch, rows, 0))
    finally:
        enc.close()
    assert data == RS.encode(sch, rows)
    dec = native.Decoder(sch, 0, **SPLITS)
    try:
        b, used = dec.decode(np.frombuffer(data, dtype=np.uint8))
        assert used == len(data) and b.info["error_code"] == 0 and b.n_rows == len(rows)
        cols = b.to_host()
        assert len(cols) == 3 and cols[1].depth == 2
        for r, row in enumerate(rows):
            assert _norm(cols[1].get(r)) == _norm(row[1]) and cols[0].get(r) == row[0]
        b.release()
    finally:
        dec.close()


@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("leaf", ROW_LEAVES)
def test_unsafe_rows_encode_sync_and_pipelined(native, leaf, nullable):
    from oracle import unsaferow
    sch = _schema(leaf, nullable)
    rows = _rows(leaf, nullable, seed=3)
    want = RS.encode(sch, rows)
    buf, offs = unsaferow.unsafe_rows(sch, rows)
    enc = native.Encoder(sch, 0, **SPLITS)
    try:
        enc.encode_rows(buf, offs)
        assert enc.result_host() == want
        subs = [enc.submit_rows(buf, offs) for _ in range(3)]
        for sub in subs:
            sub.wait()
            assert sub.result_host() == want
            sub.release()
    finally:
        enc.close()


def test_write_errors(native):
    from oracle import unsaferow
    sch = _schema("long", False)
    enc = native.Encoder(sch, 0, **SPLITS)
    try:
        with pytest.raises(native.NullPointerException) as e:
            enc.encode(A.columns_from_rows(sch, [(0, [[1]], 0.0), (1, None, 1.0)], 0))
        assert e.value.row == 1
        buf, offs = unsaferow.unsafe_rows(sch, [(0, [[1]], 0.0), (1, [[2], None, [3]], 1.0)])
        with pytest.raises(native.NullPointerException) as e:                 # a null inner array
            enc.encode_rows(buf, offs)
        assert e.value.row == 1
        cols = A.columns_from_rows(sch, [(0, [[1, 2]], 0.0), (1, [[3]], 1.0)], 0)
        cols[1].offsets[1][1] = 5                                             # row 1's inner list now has length -2
        with pytest.raises(native.TfrError) as e:
            enc.encode(cols)
        assert e.value.code == A.TFR_E_INVALID_ARG and e.value.row == 1
    finally:
        enc.close()


def _multi_tile_rows(n, seed):
    """more rows than one scan tile (2048), with nulls and empty rows in runs across the tile edges"""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        edge = min(i % 2048, 2048 - i % 2048) < 6
        k = int(rng.integers(0, 4))
        if (edge and k == 0) or i % 13 == 0:
            x = None
        elif (edge and k == 1) or i % 17 == 0:
            x = []
        elif edge and k == 2:
            x = [[]]
        else:
            x = [[int(v) for v in rng.integers(-100, 100, int(rng.integers(0, 5)))] for _ in range(int(rng.integers(1, 6)))]
        rows.append((i, x, 1.0))
    return rows


def test_multi_tile_batch_every_path(native):
    """rows across several scan tiles: the first decode (count mode), the steady-state pipelined submit and the general path
    (a mismatch forced at the end) give the restatement's rows"""
    sch = _schema("long", True)
    rows = _multi_tile_rows(9000, 2)
    data = RS.encode(sch, rows)
    arr = np.frombuffer(data, dtype=np.uint8)
    dec = native.Decoder(sch, 0, **SPLITS)
    try:
        for k in range(4):
            b = dec.submit(arr) if k >= 2 else dec.decode(arr)[0]
            assert b.info["error_code"] == 0 and b.n_rows == len(rows)
            c = b.to_host()[1]
            assert [c.get(r) for r in range(b.n_rows)] == [r[1] for r in rows]
            b.release()
        assert dec.stats()["speculative_submits"] >= 1
        bad = pyref.frame(pyref.example({"id": pyref.int64_feature(9000), "x_values": pyref.int64_feature(1),
                                         "x_row_splits": pyref.int64_feature(0, 2)}).SerializeToString())
        b, _ = dec.decode(np.frombuffer(data + bad, dtype=np.uint8))
        assert (b.info["error_code"], b.info["error_row"], b.info["error_field"]) == (A.TFR_E_BAD_NESTING, len(rows), 1)
        c = b.to_host()[1]
        assert [c.get(r) for r in range(b.n_rows)] == [r[1] for r in rows]
        b.release()
    finally:
        dec.close()


def _bad_records(seed=1, n=400):
    """Example payloads, about one in eight with disagreeing or malformed parts, and the expectation of each"""
    rng = np.random.default_rng(seed)
    i64, flt = pyref.int64_feature, pyref.float_feature
    payloads = []
    for i in range(n):
        lens = [int(x) for x in rng.integers(0, 5, int(rng.integers(0, 6)))]
        vals = [int(x) for x in rng.integers(0, 100, sum(lens))]
        spl = RS.splits(lens)
        feats = {"id": i64(i), "x_values": i64(*vals), "x_row_splits": i64(*spl), "w": flt(1.0)}
        k = int(rng.integers(0, 10)) if i > 3 else 0
        if k == 1:
            feats["x_row_splits"] = i64(*(spl + [spl[-1] + 1]))           # last entry not the values
        elif k == 2 and len(spl) > 2:
            feats["x_row_splits"] = i64(*([0, spl[-1] + 1] + spl[2:]))    # a decrease
        elif k == 3:
            del feats["x_row_splits"]                                     # one part missing
        elif k == 4:
            feats["x_row_splits"] = flt(0.0)                              # FloatList splits
        elif k == 5:
            feats["id"] = flt(1.0)                                        # a caller field's error, and a mismatch
            feats["x_row_splits"] = i64(*(spl + [99]))
        elif k == 6:
            feats["x_row_splits"] = i64()                                 # an empty splits list
        elif k == 7:
            feats["x_row_splits"] = i64(*([1] + spl[1:]))                 # first entry not 0
        payloads.append(pyref.example(feats).SerializeToString())
    return payloads


MODES = {"failfast": A.TFR_F_VERIFY_CRC, "drop": A.TFR_F_VERIFY_CRC | A.TFR_F_DROP_MALFORMED,
         "permissive": A.TFR_F_VERIFY_CRC | A.TFR_F_PERMISSIVE,
         "drop_resync": A.TFR_F_VERIFY_CRC | A.TFR_F_DROP_MALFORMED | A.TFR_F_RESYNC,
         "permissive_resync": A.TFR_F_VERIFY_CRC | A.TFR_F_PERMISSIVE | A.TFR_F_RESYNC}


@pytest.mark.parametrize("mode", sorted(MODES))
def test_read_errors_in_every_mode(native, mode):
    sch = _schema("long", True)
    payloads = _bad_records()
    exp = [RS.read(sch, p) for p in payloads]
    data = b"".join(pyref.frame(p) for p in payloads)
    dec = native.Decoder(sch, 0, flags=MODES[mode], **SPLITS)
    try:
        b, _ = dec.decode(np.frombuffer(data, dtype=np.uint8))
        info, cols = b.info, b.to_host()
        bad = [(i, e[1]) for i, e in enumerate(exp) if e[1] is not None]
        assert bad, "the corpus must hold failing records"
        if mode == "failfast":
            i, (code, field) = bad[0]
            assert (info["error_code"], info["error_row"], info["error_field"]) == (code, i, field)
            kept = list(range(i))
        else:
            assert [(d[0], d[2], d[3]) for d in b.dropped()] == [(i, c, f) for i, (c, f) in bad]
            kept = [i for i, e in enumerate(exp) if e[1] is None]
        if mode.startswith("permissive"):
            assert b.n_rows == len(payloads)
            for r in range(len(payloads)):
                assert cols[1].get(r) == (exp[r][0][1] if exp[r][1] is None else None)
        else:
            assert b.n_rows == len(kept)
            for r, i in enumerate(kept):
                assert cols[1].get(r) == exp[i][0][1] and cols[0].get(r) == exp[i][0][0]
        b.release()
    finally:
        dec.close()


def _stream(native, sch, data, flags, seed, **kw):
    """data read in random blocks (the carry of each goes into the next): the delivered rows of column 1 and of the row-index
    column, and the dropped list"""
    rng = np.random.default_rng(seed)
    dec = native.Decoder(sch, 0, flags=flags, **SPLITS, **kw)
    got, idx, dropped, pos, base, entry, offset = [], [], [], 0, 0, 0, 0
    try:
        while pos < len(data):
            end = min(len(data), pos + int(rng.integers(1, 40000)))
            final = end == len(data)
            b, used = dec.decode(np.frombuffer(data[pos:end], dtype=np.uint8), is_final=final, first_entry=entry, first_offset=pos)
            cols = b.to_host()
            got += [cols[1].get(r) for r in range(b.n_rows)]
            idx += [(cols[3].get(r), cols[4].get(r)) for r in range(b.n_rows)]
            dropped += [(base + d[0], d[2], d[3]) for d in b.dropped()]
            ext = b.extent()[1]
            base += ext
            entry += ext
            b.release()
            if used == 0 and not final:
                continue
            pos += used
            if final:
                break
        return got, idx, dropped
    finally:
        dec.close()


@pytest.mark.parametrize("mode", ["drop", "drop_resync", "permissive", "permissive_resync"])
def test_random_block_cuts_with_row_index(native, mode):
    from spark_tfrecord_b200 import io
    sch = _schema("long", True)
    rsch = StructType(list(sch.fields) + [StructField("_tmp_metadata_row_index", LongType(), False),
                                          StructField("_tmp_metadata_record_offset", LongType(), False)])
    payloads = _bad_records(seed=5)
    exp = [RS.read(sch, p) for p in payloads]
    frames = [pyref.frame(p) for p in payloads]
    starts = np.concatenate([[0], np.cumsum([len(f) for f in frames])[:-1]]).tolist()
    data = b"".join(frames)
    for seed in range(3):
        got, idx, dropped = _stream(native, io._decoder_schema(rsch), data, MODES[mode], seed)
        assert dropped == [(i, e[1][0], e[1][1]) for i, e in enumerate(exp) if e[1] is not None]
        if mode.startswith("permissive"):
            assert got == [e[0][1] if e[1] is None else None for e in exp]
            assert idx == [(i, starts[i]) for i in range(len(exp))]
        else:
            assert got == [e[0][1] for e in exp if e[1] is None]
            assert idx == [(i, starts[i]) for i, e in enumerate(exp) if e[1] is None]


def _clean(n, seed, big=False):
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        k = 3000 if big else 4
        rows.append((i, [[int(x) for x in rng.integers(-2**40, 2**40, int(rng.integers(0, 2 * k)))] for _ in range(int(rng.integers(1, 4)))],
                     1.0))
    return rows


@pytest.mark.parametrize("big", [False, True])
def test_fast_path_hands_a_mismatch_to_the_general_path(native, big):
    """a batch whose only failing row is a splits mismatch, on the tile path and (records larger than a tile) the large-record
    path: the fast kernel cannot see it, the assembly's verdict sends the batch to the general path, and the result is exact"""
    sch = _schema("long", True)
    rows = _clean(400 if not big else 60, 7, big)
    low = RS.lowered_schema(sch)
    payloads = [pyref.frame(pyref.serialize_example_bytes(low, RS.lower_row(sch, r))) for r in rows]
    bad_at = len(rows) // 2
    lr = RS.lower_row(sch, rows[bad_at])
    lr = lr[:3] + ([0] + [x + 1 for x in lr[3][1:]],)                     # the last entry no longer the number of values
    payloads[bad_at] = pyref.frame(pyref.serialize_example_bytes(low, lr))
    data = b"".join(payloads)
    clean = RS.encode(sch, rows)
    dec = native.Decoder(sch, 0, **SPLITS)
    try:
        for _ in range(2):                                                # the clean file: the fast path takes it
            b, _ = dec.decode(np.frombuffer(clean, dtype=np.uint8))
            assert b.info["error_code"] == 0 and [b.to_host()[1].get(r) for r in range(b.n_rows)] == [r[1] for r in rows]
            b.release()
        st0 = dec.stats()
        assert st0["general_path_batches"] == 0 and (st0["large_record_batches"] > 0) == big
        b, _ = dec.decode(np.frombuffer(data, dtype=np.uint8))
        info = b.info
        assert (info["error_code"], info["error_row"], info["error_field"]) == (A.TFR_E_BAD_NESTING, bad_at, 1)
        assert [b.to_host()[1].get(r) for r in range(b.n_rows)] == [r[1] for r in rows[:bad_at]]
        assert dec.stats()["general_path_batches"] == st0["general_path_batches"] + 1
        b.release()
    finally:
        dec.close()


def test_pipelined_submit_takes_no_extra_synchronisation(native):
    """the same rows submitted to a splits decoder and to a lengths decoder: the same number of batches stay speculative (no
    host synchronisation) and none is redone; the columns equal the restatement"""
    sch = _schema("long", True)
    rows = _clean(20000, 11)
    stats = []
    for splits in (True, False):
        data = np.frombuffer((RS if splits else RR).encode(sch, rows), dtype=np.uint8)
        dec = native.Decoder(sch, 0, ragged=True, row_splits=splits)
        try:
            for k in range(8):
                b = dec.submit(data)
                if k == 7:
                    c = b.to_host()[1]
                    assert [c.get(r) for r in range(b.n_rows)] == [r[1] for r in rows]
                b.release()
            st = dec.stats()
            stats.append((st["speculative_submits"], st["speculative_redone"], st["general_path_batches"]))
        finally:
            dec.close()
    assert stats[0] == stats[1] and stats[0][0] > 0 and stats[0][1] == 0


def test_views_arrow_rows_partition_async(native):
    import pyarrow as pa
    import partition_rows as PR
    import unsafe_row_reader as UR
    sch = _schema("string", True)
    rows = _rows("string", True, n=120, seed=9)
    data = np.frombuffer(RS.encode(sch, rows), dtype=np.uint8)
    dec = native.Decoder(sch, 0, **SPLITS)
    try:
        for submit in (False, True, True):
            b = dec.submit(data) if submit else dec.decode(data)[0]
            b.wait()
            arrs = b.to_arrow()
            assert pa.types.is_list(arrs[1].type) and pa.types.is_list(arrs[1].type.value_type)
            assert arrs[1].to_pylist() == [r[1] for r in rows]
            c = b.device_columns()[1]                                 # the device view
            assert c.n_offsets[0] == len(rows) + 1 and c.n_offsets[1] == sum(len(r[1]) for r in rows if r[1] is not None) + 1
            want = [UR.normalise(sch, r) for r in rows]
            h, o = b.unsafe_rows()
            assert UR.read_rows(sch, h, o) == want
            b.release()
        ptypes, pvals = ["string", "int"], ["p=1", 7]
        for asy in (False, True):
            b, _ = dec.decode(data)
            part = (PR.partition_row(ptypes, pvals), PR.var_flags(ptypes))
            if asy:
                b.unsafe_rows_async(to_host=True, partition=part)
            h, o = b.unsafe_rows(partition=part)
            jb, jo = PR.joined_rows(sch, [tuple(r) for r in rows], ptypes, pvals)
            assert h.tobytes() == jb.tobytes() and list(o) == list(jo)
            b.release()
    finally:
        dec.close()


def test_cross_partition_reads_fail(native):
    """a lengths file read with rowSplits and a splits file read with rowLengths: TFR_E_BAD_NESTING at x, never a misread"""
    sch = _schema("long", True)
    rows = _clean(50, 3)
    for reader_splits, data in ((True, RR.encode(sch, rows)), (False, RS.encode(sch, rows))):
        dec = native.Decoder(sch, 0, ragged=True, row_splits=reader_splits)
        try:
            b, _ = dec.decode(np.frombuffer(data, dtype=np.uint8))
            assert (b.info["error_code"], b.info["error_row"], b.info["error_field"]) == (A.TFR_E_BAD_NESTING, 0, 1)
            b.release()
        finally:
            dec.close()


def test_default_source_round_trip(native, tmp_path):
    from spark_tfrecord_b200 import io
    sch = _schema("long", True)
    rows = _rows("long", True, n=50)
    opts = {"nestedArrayFormat": "ragged", "raggedPartition": "rowSplits"}
    path = str(tmp_path / "part-0.tfrecord")
    w = io.DefaultSource().prepareWrite(opts, sch).newInstance(path, sch)
    for r in rows:
        w.write(r)
    w.close()
    assert open(path, "rb").read() == RS.encode(sch, rows)
    got = list(io.DefaultSource().buildReader(sch, sch, opts)(io.PartitionedFile(path)))
    assert [tuple(r) for r in got] == [tuple(r) for r in rows]
    inferred = io.DefaultSource().inferSchema(opts, [path])
    assert sorted(f.name for f in inferred.fields) == ["id", "w", "x_row_splits", "x_values"]
