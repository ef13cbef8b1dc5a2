"""GPU tests of PERMISSIVE (TFR_F_PERMISSIVE, Spark's mode=PERMISSIVE): a record that fails is read as a row of nulls at
its own position, its payload in the corrupt-record column; a framing error still ends the block.

The expectation comes from the oracle alone.  test_gpu_drop_malformed.expected decodes the block with every failing
record cut out, for the schema without the corrupt-record column; then a null row goes in at each cut frame's index, and
the corrupt-record column is built from those frames' payloads (data[off + 12 : end - 4]).  The batch must then have
  * every column, bit for bit, null counts included;
  * tfr_batch_info: n_rows = kept + corrupt rows, error_row == n_rows on a framing error, the rest as in drop mode;
  * tfr_batch_dropped's list, unchanged from drop mode, and counter [10];
  * UnsafeRows (tfr_batch_rows, _with_partition, _async; host and device) equal to oracle.unsaferow's rows of those columns.
The corrupt-record column goes first, in the middle and last, or is left out (rows of nulls only)."""
import os
import random

import numpy as np
import pytest

import test_gpu_drop_malformed as D
import wire_rewrite as W
from oracle import corpus, pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200._cabi import HostColumn
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_decode_rows import _schema_of_case
from util import assert_columns_equal, record_offsets

pytestmark = pytest.mark.gpu

PERM = A.TFR_F_DEFAULT | A.TFR_F_PERMISSIVE
CORRUPT = "_corrupt_record"
POSITIONS = ["first", "middle", "last", None]


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def with_corrupt(sch, pos):
    """(the schema with the corrupt-record column at `pos`, its index); pos None: (sch, None)"""
    if pos is None:
        return sch, None
    fields = list(sch.fields)
    at = {"first": 0, "middle": len(fields) // 2, "last": len(fields)}[pos]
    fields.insert(at, StructField(CORRUPT, BinaryType()))
    return StructType(fields), at


def expand(col, bad, n_total):
    """`col` of the kept rows with a null, empty row at each index of `bad` (sorted output rows)"""
    keep = np.ones(n_total, bool)
    keep[bad] = False
    idx = np.nonzero(keep)[0]
    bits = np.ones(col.n_rows, np.uint8) if col.validity is None else np.unpackbits(col.validity, bitorder="little")[:col.n_rows]
    nv = np.zeros(n_total, np.uint8)
    nv[idx] = bits
    offsets = [o.copy() for o in col.offsets]
    values = col.values
    if col.n_levels:
        bb = np.searchsorted(np.asarray(bad, np.int64), np.arange(n_total + 1), side="left")
        offsets[0] = col.offsets[0][np.arange(n_total + 1) - bb]
    elif col.elem_type != TFR_T_NULL:
        values = np.zeros(n_total, col.values.dtype)
        values[idx] = col.values[:col.n_rows]
    return HostColumn(col.elem_type, col.depth, n_total, np.packbits(nv, bitorder="little"), offsets, values)


def corrupt_column(data, dropped, n_total):
    bad = [i for i, _, _, _ in dropped]
    offs = record_offsets(bytes(data))
    payloads = [bytes(data[int(offs[i]) + 12:int(offs[i + 1]) - 4]) for i in bad]
    bits = np.zeros(n_total, np.uint8)
    bits[bad] = 1
    cum = np.concatenate([[0], np.cumsum([len(p) for p in payloads], dtype=np.int64)]).astype(np.int32)
    bb = np.searchsorted(np.asarray(bad, np.int64), np.arange(n_total + 1), side="left")
    vals = np.frombuffer(b"".join(payloads), np.uint8) if payloads else np.zeros(0, np.uint8)
    return HostColumn(TFR_T_BINARY, 0, n_total, np.packbits(bits, bitorder="little"), [cum[bb]], vals)


def expected(oracle, data, sch, rt, flags, cf, is_final=True) -> D.Expect:
    """PERMISSIVE's expectation for schema `sch` (its corrupt-record column at index cf, or None) from drop mode's"""
    sub = sch if cf is None else StructType([f for i, f in enumerate(sch.fields) if i != cf])
    e = D.expected(oracle, data, sub, rt, (flags & ~A.TFR_F_PERMISSIVE) | A.TFR_F_DROP_MALFORMED, is_final)
    bad = [i for i, _, _, _ in e.dropped]
    n_total = e.info["n_rows"] + len(bad)
    cols = [expand(c, bad, n_total) for c in e.columns]
    if cf is not None:
        cols.insert(cf, corrupt_column(data, e.dropped, n_total))
    info = dict(e.info, n_rows=n_total)
    if info["error_code"]:
        assert info["error_row"] == n_total, info
    # drop mode's list, its schema fields numbered in `sch` (the corrupt-record column is never the failing field)
    dropped = [(i, off, code, f + (cf is not None and f >= cf)) for i, off, code, f in e.dropped]
    return D.Expect(cols, info, dropped)


def check_fresh(native, oracle, data, sch, rt, pos, flags=PERM, is_final=True, what=""):
    """fresh PERMISSIVE decoders, the corrupt-record column at `pos`: info, list, columns, counter [10], sync rows, rows with
    a partition row"""
    full, cf = with_corrupt(sch, pos)
    exp = expected(oracle, data, full, rt, flags, cf, is_final)
    what = f"{what} (corrupt column {pos})"
    for part in (None, D.PART):
        dec = native.Decoder(full, rt, flags=flags, corrupt_field=cf)
        b, used = dec.decode(data, is_final=is_final)
        assert used == exp.info["consumed_bytes"], what
        D.check_info(b, exp, what)
        if part is None:
            assert_columns_equal(b.to_host(), exp.columns, None, what)
            st = dec.stats()
            assert st["records_corrupt"] == len(exp.dropped) and st["records_dropped"] == 0, (what, st)
        D.check_rows(b, full, exp, part, what)
        b.release()
        dec.close()
    return exp


# ---------------------------------------------------------------------------------------------
# 1. every case and golden vector
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pos", POSITIONS)
def test_every_case(native, oracle, pos):
    import cases as CS
    n = bad = 0
    for c in CS.all_cases():
        if c.record_type == TFR_RT_BYTE_ARRAY:
            continue
        exp = check_fresh(native, oracle, c.data(), _schema_of_case(c), c.record_type, pos,
                          getattr(c, "flags", A.TFR_F_DEFAULT) | A.TFR_F_PERMISSIVE, getattr(c, "is_final", True), what=c.name)
        n += 1
        bad += len(exp.dropped)
    assert n > 20 and bad > 10, (n, bad)


@pytest.mark.parametrize("pos", POSITIONS)
def test_golden_vectors(native, oracle, pos):
    import test_golden as G
    bad = 0
    for e in G.INDEX:
        if e["record_type"] == 2:
            continue
        data = open(os.path.join(G.HERE, e["file"]), "rb").read()
        exp = check_fresh(native, oracle, data, G.schema_of(e), e["record_type"], pos, e["flags"] | A.TFR_F_PERMISSIVE, e["is_final"],
                          what=e["name"])
        bad += len(exp.dropped)
    assert bad > 5


# ---------------------------------------------------------------------------------------------
# 2. seeded corpora, a fresh decoder
# ---------------------------------------------------------------------------------------------
CORPORA = ["cfg2", "ragged_strings", "sequence_example", "w130_general"]


@pytest.mark.parametrize("lencrc", [False, True], ids=["clean_tail", "lencrc_flip"])
@pytest.mark.parametrize("name", CORPORA)
def test_corpus_fresh_decoder(native, oracle, name, lencrc):
    n = 600 if name == "w130_general" else 1500
    for seed, pos in ((1, "middle"), (2, "first"), (3, None)):
        sch, rt, rows, frames, data = D.bad_block(name, n, seed * 101 + len(name), 9, lencrc)
        exp = check_fresh(native, oracle, data, sch, rt, pos, what=f"{name} seed {seed}")
        assert len(exp.dropped) >= 5, exp.dropped
        assert bool(exp.info["error_code"]) == lencrc, exp.info
        if lencrc:
            assert exp.info["error_code"] == A.TFR_E_CRC_LENGTH and exp.info["error_row"] == exp.info["n_rows"]


# ---------------------------------------------------------------------------------------------
# 3. a decoder in its pipelined steady state: clean, bad, clean
# ---------------------------------------------------------------------------------------------
def null_column(n):
    return HostColumn(TFR_T_BINARY, 0, n, np.zeros((n + 7) // 8, np.uint8), [np.zeros(n + 1, np.int32)], np.zeros(0, np.uint8))


@pytest.mark.parametrize("name", CORPORA)
def test_corpus_pipelined(native, oracle, name):
    n = 600 if name == "w130_general" else 1500
    sch, rt, rows, frames, data = D.bad_block(name, n, 7 + len(name), 6)
    full, cf = with_corrupt(sch, "last")
    clean = b"".join(frames)
    want_clean = expected(oracle, clean, full, rt, PERM, cf)
    exp = expected(oracle, data, full, rt, PERM, cf)
    assert len(exp.dropped) >= 3
    dec = native.Decoder(full, rt, flags=PERM, corrupt_field=cf)
    ff = native.Decoder(sch, rt, flags=A.TFR_F_DEFAULT)
    for _ in range(3):                                         # learning
        b = dec.submit(clean)
        D.check_info(b, want_clean, f"{name} learning")
        b.release()
    pipelined = name in D.PIPELINED

    def clean_batch(tag):
        s0 = dec.stats()
        b = dec.submit(clean)
        b.unsafe_rows_async(True)
        D.check_info(b, want_clean, tag)
        got = b.to_host()
        assert_columns_equal(got, want_clean.columns, None, tag)
        D.check_rows(b, full, want_clean, None, tag)
        b.release()
        d = D.delta(s0, dec.stats())
        if pipelined:
            assert d["speculative_submits"] == 1 and d["speculative_redone"] == 0, (tag, d)
        assert d["records_corrupt"] == 0, (tag, d)
        return got

    got = clean_batch(f"{name} clean before")
    bf, _ = ff.decode(clean)                                  # a clean block: FAILFAST's columns and an all-null corrupt column
    want = bf.to_host()
    want.insert(cf, null_column(bf.n_rows))
    assert_columns_equal(got, want, None, f"{name} clean vs FAILFAST")
    bf.release()
    s0 = dec.stats()
    b = dec.submit(data)
    b.unsafe_rows_async(True)
    D.check_info(b, exp, f"{name} bad")
    assert_columns_equal(b.to_host(), exp.columns, None, f"{name} bad")
    D.check_rows(b, full, exp, None, f"{name} bad (async)")
    b.release()
    d = D.delta(s0, dec.stats())
    assert d["records_corrupt"] == len(exp.dropped) and d["records_dropped"] == 0, d
    if pipelined:
        assert d["speculative_submits"] == 1 and d["speculative_redone"] == 1, d
    clean_batch(f"{name} clean after")
    b = dec.submit(data)                                      # a pipelined bad block whose rows come with a partition row
    b.unsafe_rows_async(True, (D.P.partition_row(*D.PART), D.P.var_flags(D.PART[0])))
    D.check_info(b, exp, f"{name} bad, partitioned")
    D.check_rows(b, full, exp, D.PART, f"{name} bad (async, partitioned)")
    b.release()
    clean_batch(f"{name} clean at the end")
    dec.close()
    ff.close()


# ---------------------------------------------------------------------------------------------
# 4. streamed in 1 MiB blocks with carry-over
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lencrc", [False, True], ids=["clean_tail", "lencrc_flip"])
@pytest.mark.parametrize("name", ["cfg2", "ragged_strings"])
def test_corpus_streamed(native, oracle, name, lencrc):
    n = {"cfg2": 3000, "ragged_strings": 30000}[name]
    sch, rt, rows, frames, data = D.bad_block(name, n, 31 + len(name), 40, lencrc)
    full, cf = with_corrupt(sch, "middle")
    dec = native.Decoder(full, rt, flags=PERM, corrupt_field=cf)
    ff = native.Decoder(sch, rt, flags=A.TFR_F_DEFAULT)
    warm = b"".join(frames)[:1 << 20]
    for d_ in (dec, ff):                                      # both in their steady state: the blocks are submitted pipelined
        for _ in range(3):
            d_.submit(warm, is_final=False).release()
    pos, blocks, bad, stopped = 0, 0, 0, False
    while True:
        chunk = data[pos:pos + (1 << 20)]
        final = pos + len(chunk) >= len(data)
        exp = expected(oracle, chunk, full, rt, PERM, cf, is_final=final)
        b = dec.submit(chunk, is_final=final)
        bf = ff.submit(chunk, is_final=final)
        used = b.consumed()
        assert used == bf.consumed(), (blocks, used, bf.consumed())
        bf.release()
        D.check_info(b, exp, f"{name} block {blocks}")
        assert_columns_equal(b.to_host(), exp.columns, None, f"{name} block {blocks}")
        b.release()
        bad += len(exp.dropped)
        blocks += 1
        if exp.info["error_code"]:
            stopped = True
            break
        pos += used
        if final:
            break
    assert blocks >= 3 and bad >= 10 and stopped == lencrc, (blocks, bad, stopped)
    assert dec.stats()["records_corrupt"] == bad
    dec.close()
    ff.close()


# ---------------------------------------------------------------------------------------------
# 5. edge cases
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pos", ["first", None])
def test_every_record_bad(native, oracle, pos):
    sch, rt, rows, frames = D.cfg2_corpus(200, 5)
    data = b"".join(bytes(f[:-1]) + bytes([f[-1] ^ 0x10]) for f in frames)   # every payload CRC wrong
    exp = check_fresh(native, oracle, data, sch, rt, pos, what="all bad")
    assert exp.info["n_rows"] == 200 and len(exp.dropped) == 200
    full, cf = with_corrupt(sch, pos)
    dec = native.Decoder(full, rt, flags=PERM, corrupt_field=cf)
    b, _ = dec.decode(data)
    cols = b.to_host()
    assert all(c.null_count == 200 for i, c in enumerate(cols) if i != cf)
    if cf is not None:
        assert cols[cf].null_count == 0 and [cols[cf].get(r) for r in range(200)] == [f[12:-4] for f in frames]
    b.release()
    dec.close()


def test_verify_crc_off(native, oracle):
    """without TFR_F_VERIFY_CRC a payload bit flip is not a record error (unless it breaks the protobuf)"""
    sch, rt, rows, frames = D.cfg2_corpus(800, 9)
    R_ = random.Random(9)
    data = D.corrupt(frames, sch, rows, rt, R_, sorted(R_.sample(range(800), 12)))
    exp = check_fresh(native, oracle, data, sch, rt, "middle", flags=A.TFR_F_PERMISSIVE, what="verify off")
    full, cf = with_corrupt(sch, "middle")
    with_crc = expected(oracle, data, full, rt, PERM, cf)
    assert len(exp.dropped) < len(with_crc.dropped)
    assert all(code != A.TFR_E_CRC_DATA for _, _, code, _ in exp.dropped)


@pytest.mark.parametrize("kind", [BinaryType(), LongType(), ArrayType(FloatType())])
def test_a_feature_named_like_the_corrupt_column(native, oracle, kind):
    """records that carry a feature of the corrupt column's name: PERMISSIVE ignores it (a wrong kind is no kind mismatch);
    FAILFAST with the same schema reads it as an ordinary BinaryType feature"""
    base, _ = corpus.cfg2_columns(300, seed=17)
    R_ = np.random.default_rng(17)
    enc = StructType(list(base.fields) + [StructField(CORRUPT, kind)])
    val = {"BinaryType": lambda: R_.integers(0, 256, int(R_.integers(0, 40)), dtype=np.uint8).tobytes(),
           "LongType": lambda: int(R_.integers(-1000, 1000)),
           "ArrayType": lambda: [float(x) for x in R_.random(3).astype(np.float32)]}[type(kind).__name__]
    _, cols = corpus.cfg2_columns(300, seed=17)
    rows = [tuple(c.get(r) for c in cols) + (val(),) for r in range(300)]
    frames = [pyref.frame_fast(W.canonical(enc, row)) for row in rows]
    frames[40] = frames[40][:-1] + bytes([frames[40][-1] ^ 1])         # one payload CRC failure
    data = b"".join(frames)
    full = StructType(list(base.fields) + [StructField(CORRUPT, BinaryType())])
    cf = len(base.fields)
    exp = expected(oracle, data, full, TFR_RT_EXAMPLE, PERM, cf)
    assert [i for i, _, _, _ in exp.dropped] == [40]
    dec = native.Decoder(full, TFR_RT_EXAMPLE, flags=PERM, corrupt_field=cf)
    b, _ = dec.decode(data)
    D.check_info(b, exp, "permissive")
    got = b.to_host()
    assert_columns_equal(got, exp.columns, None, "permissive")
    assert got[cf].null_count == 299 and got[cf].get(40) == frames[40][12:-4]
    b.release()
    dec.close()
    want = oracle.decode(data, full, TFR_RT_EXAMPLE)
    dec = native.Decoder(full, TFR_RT_EXAMPLE)
    b, _ = dec.decode(data)
    assert {k: b.info[k] for k in ("n_rows", "error_code", "error_row", "error_field")} == \
        {k: want.info[k] for k in ("n_rows", "error_code", "error_row", "error_field")}
    if isinstance(kind, BinaryType):
        assert b.info["error_code"] == A.TFR_E_CRC_DATA and b.info["n_rows"] == 40
    else:
        assert b.info["error_code"] == A.TFR_E_KIND_MISMATCH and b.info["error_row"] == 0
    assert_columns_equal(b.to_host(), want.columns, None, "failfast")
    b.release()
    dec.close()


def test_decimal_schema(native, oracle):
    """columns are right; UnsafeRows of a DecimalType schema are refused as without the flag"""
    sch = StructType([StructField("d", DecimalType()), StructField("s", StringType())])
    clean, rc, _ = oracle.encode(A.columns_from_rows(sch, [(float(i) / 4, f"r{i}") for i in range(100)]), sch)
    assert rc == 0
    offs = record_offsets(clean)
    frames = [bytes(clean[int(offs[i]):int(offs[i + 1])]) for i in range(100)]
    for i in (3, 50):
        frames[i] = frames[i][:-1] + bytes([frames[i][-1] ^ 4])
    data = b"".join(frames)
    full, cf = with_corrupt(sch, "middle")
    exp = check_fresh(native, oracle, data, sch, TFR_RT_EXAMPLE, "middle", what="decimal")
    assert [i for i, _, _, _ in exp.dropped] == [3, 50]
    dec = native.Decoder(full, TFR_RT_EXAMPLE, flags=PERM, corrupt_field=cf)
    b, _ = dec.decode(data)
    with pytest.raises(native.TfrError) as ei:
        b.unsafe_rows(True)
    assert ei.value.code == A.TFR_E_UNSUPPORTED_TYPE
    b.release()
    dec.close()


def test_default_source_load(native, oracle, tmp_path):
    from spark_tfrecord_b200.io import DefaultSource, PartitionedFile, TFRecordFileReader
    sch, rt, rows, frames, data = D.bad_block("ragged_strings", 700, 13, 7)
    path = tmp_path / "part-00000.tfrecord"
    path.write_bytes(data)
    full, cf = with_corrupt(sch, "last")
    exp = expected(oracle, data, full, rt, PERM, cf)
    want = [tuple(c.get(r) for c in exp.columns) for r in range(exp.info["n_rows"])]
    assert sum(r[cf] is not None for r in want) == len(exp.dropped) >= 5
    for mode in ("PERMISSIVE", "permissive"):
        assert DefaultSource().load(str(tmp_path), full, {"mode": mode}) == want
    got = list(TFRecordFileReader.readFile(None, {"mode": "PERMISSIVE"}, PartitionedFile(str(path)), full, block_bytes=64 << 10))
    assert got == want
    # the corrupt column pruned by a projection: rows of None at the failing records
    pruned = expected(oracle, data, sch, rt, PERM, None)
    want_pruned = [tuple(c.get(r) for c in pruned.columns) for r in range(pruned.info["n_rows"])]
    assert want_pruned == [r[:cf] for r in want]
    bad = {i for i, _, _, _ in exp.dropped}
    assert all(all(v is None for v in want_pruned[i]) for i in bad)
    reader = DefaultSource().buildReader(full, sch, {"mode": "PERMISSIVE"})
    assert list(reader(PartitionedFile(str(path)))) == want_pruned
    got = list(TFRecordFileReader.readFile(None, {"mode": "PERMISSIVE"}, PartitionedFile(str(path)), sch, block_bytes=64 << 10,
                                           dataSchema=full))
    assert got == want_pruned
