"""GPU tests of drop mode (TFR_F_DROP_MALFORMED, Spark's mode=DROPMALFORMED): a record that fails is dropped and the block
is decoded on; a framing error still ends the block.

The expectation comes from the oracle alone (`expected`): decode the block with oracle.decode; on a record error at row e,
note (frame index, offset, code, field), cut that frame out of the block (util.record_offsets) and decode again, until
the oracle reports no record error.  The batch must then have
  * every column, bit for bit, of the oracle's decode of the kept frames, null counts included;
  * tfr_batch_info: n_rows the kept rows, n_records the frames in the consumed bytes (dropped ones included),
    consumed_bytes the framing outcome, and error_code / error_row / error_field only for a framing error, error_row
    being the frame index at which framing stopped;
  * tfr_batch_dropped's list, in record order;
  * UnsafeRows (tfr_batch_rows, _with_partition, _async; host and device) equal to oracle.unsaferow's rows of those columns.
Blocks: every case of tests/cases.py and every golden vector; seeded corpora with bad records at random positions
(wire_rewrite.error_record's CRC-valid error classes and payload bit flips, then optionally a length-CRC flip after the
drops) of configs[1]-shaped Examples, ragged strings, SequenceExamples, ByteArray rows and a 130-field schema (general
path).  Each is decoded by a fresh decoder, by a decoder in its pipelined steady state (a bad block between clean ones,
counters [1] speculative submits, [2] redone, [9] records dropped), and streamed in 1 MiB blocks with carry-over, where
every block's tfr_batch_consumed equals a FAILFAST decoder's on the same bytes."""
import os
import random

import numpy as np
import pytest

import partition_rows as P
import wire_rewrite as W
from oracle import corpus, pyref
from oracle import unsaferow as U
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_decode_rows import _Dev, _has_decimal, _schema_of_case
from test_gpu_encode_rows import rows_of
from util import assert_columns_equal, record_offsets
import unsafe_row_reader as R

pytestmark = pytest.mark.gpu

DROP = A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED
PART = (["string", "int"], ["2024-05-01", 17])
ERROR_CLASSES = ["kind_mismatch", "kind_not_set", "empty_scalar", "null_in_nonnull", "bad_nesting", "malformed", "crc"]


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def delta(s0, s1):
    return {k: s1[k] - s0[k] for k in s0}


class Expect:
    def __init__(self, columns, info, dropped):
        self.columns, self.info, self.dropped = columns, info, dropped


def expected(oracle, data, sch, rt, flags, is_final=True) -> Expect:
    """the oracle's decode of `data` with every failing record cut out, one at a time (see the module docstring)"""
    buf = bytes(data)
    offs = record_offsets(buf)
    cur = [(i, int(offs[i]), int(offs[i + 1])) for i in range(len(offs) - 1)]
    tail = buf[int(offs[-1]):]
    dropped, dbytes = [], 0
    oflags = flags & ~A.TFR_F_DROP_MALFORMED
    while True:
        r = oracle.decode(b"".join(buf[a:b] for _, a, b in cur) + tail, sch, rt, flags=oflags, is_final=is_final)
        code = r.info["error_code"]
        if code not in A.RECORD_ERRORS:
            break
        i, a, b = cur.pop(r.info["error_row"])
        dropped.append((i, a, code, r.info["error_field"]))
        dbytes += b - a
    nd = len(dropped)
    info = {"n_rows": r.info["n_rows"], "n_records": r.info["n_records"] + nd, "consumed_bytes": r.info["consumed_bytes"] + dbytes,
            "error_code": code, "error_row": r.info["error_row"] + nd if code else -1, "error_field": r.info["error_field"] if code else -1}
    return Expect(r.columns, info, dropped)


def check_info(batch, exp: Expect, what=""):
    got = {k: batch.info[k] for k in exp.info}
    assert got == exp.info, f"{what}: info {got} != {exp.info}"
    assert batch.dropped() == exp.dropped, f"{what}: dropped {batch.dropped()} != {exp.dropped}"
    assert batch.consumed() == exp.info["consumed_bytes"], what


def want_rows(sch, exp: Expect, part=None):
    rows = rows_of(exp.columns, exp.info["n_rows"])
    if part is None:
        data, offs = U.unsafe_rows(sch, rows)
        return data, offs.astype(np.int64)
    return P.joined_rows(sch, rows, *part)


def device_rows(batch, part):
    import torch
    rp, op, n, nb = batch.unsafe_rows(False, part)
    offs = torch.as_tensor(_Dev(op, n + 1, "<i8"), device="cuda").cpu().numpy()
    rows = torch.as_tensor(_Dev(rp, nb, "|u1"), device="cuda").cpu().numpy() if nb else np.zeros(0, np.uint8)
    return rows, offs


def assert_rows(sch, got, want, what):
    (gr, go), (wr, wo) = got, want
    assert np.array_equal(go, wo) and np.array_equal(gr, wr), f"{what}: {R.first_diff(sch, gr, go, wr, wo)}"


def check_rows(batch, sch, exp: Expect, part=None, what=""):
    """host and device UnsafeRows of `batch` (with `part`: (partition types, values) appended)"""
    if _has_decimal(sch):
        return
    w = want_rows(sch, exp, part)
    pr = None if part is None else (P.partition_row(*part), P.var_flags(part[0]))
    hr, ho = batch.unsafe_rows(True, pr)
    assert_rows(sch, (hr.copy(), ho.copy()), w, f"{what} host rows")
    assert_rows(sch, device_rows(batch, pr), w, f"{what} device rows")


def check_fresh(native, oracle, data, sch, rt, flags=DROP, is_final=True, what="", exp=None):
    """a fresh drop-mode decoder: info, dropped list, columns, sync rows; a second one: partition rows"""
    exp = exp or expected(oracle, data, sch, rt, flags, is_final)
    for part in (None, PART):
        dec = native.Decoder(sch, rt, flags=flags)
        b, used = dec.decode(data, is_final=is_final)
        assert used == exp.info["consumed_bytes"], what
        check_info(b, exp, what)
        if part is None:
            assert_columns_equal(b.to_host(), exp.columns, None, what)
            assert dec.stats()["records_dropped"] == len(exp.dropped), what
        check_rows(b, sch, exp, part, what)
        b.release()
        dec.close()
    return exp


# ---------------------------------------------------------------------------------------------
# corpora
# ---------------------------------------------------------------------------------------------
def corrupt(frames, sch, rows, rt, R_, bad, lencrc_at=None):
    """frames with a failing record at each index of `bad` (an error_record class, or a payload bit flip) and, with
    `lencrc_at`, a flipped length-CRC bit in that frame (a framing error)"""
    frames = list(frames)
    for i in bad:
        cls = R_.choice(ERROR_CLASSES) if rt != TFR_RT_BYTE_ARRAY else "crc"
        e = None if cls == "crc" else W.error_record(sch, rows[i], rt, cls, R_)
        if e is not None and e[1] != 0:
            frames[i] = pyref.frame_fast(e[0])
            continue
        fr = bytearray(frames[i])
        if len(fr) <= 16:
            continue
        fr[12 + R_.randrange(len(fr) - 16)] ^= 1 << R_.randrange(8)
        frames[i] = bytes(fr)
    if lencrc_at is not None:
        fr = bytearray(frames[lencrc_at])
        fr[8 + R_.randrange(4)] ^= 1 << R_.randrange(8)
        frames[lencrc_at] = bytes(fr)
    return b"".join(frames)


def cfg2_corpus(n, seed):
    sch, cols = corpus.cfg2_columns(n, seed=seed)
    rows = [tuple(c.get(r) for c in cols) for r in range(n)]
    return sch, TFR_RT_EXAMPLE, rows, [pyref.frame_fast(W.canonical(sch, row)) for row in rows]


def wire_corpus(n, seed, width, rt, **kw):
    sch, gen = W.make_schema(seed, width, rt, **kw)
    r = np.random.default_rng(seed + 1)
    rows = [gen(r) for _ in range(n)]
    return sch, rt, rows, [pyref.frame_fast(W.canonical(sch, row, rt)) for row in rows]


def bytes_corpus(n, seed):
    r = np.random.default_rng(seed)
    rows = [(r.integers(0, 256, int(r.integers(1, 400)), dtype=np.uint8).tobytes(),) for _ in range(n)]
    return byte_array_schema(), TFR_RT_BYTE_ARRAY, rows, [pyref.frame_fast(row[0]) for row in rows]


CORPORA = {
    "cfg2": lambda n, s: cfg2_corpus(n, s),
    "ragged_strings": lambda n, s: wire_corpus(n, s, 12, TFR_RT_EXAMPLE),
    "sequence_example": lambda n, s: wire_corpus(n, s, 12, TFR_RT_SEQUENCE_EXAMPLE, flist_numeric=True),
    "byte_array": lambda n, s: bytes_corpus(n, s),
    "w130_general": lambda n, s: wire_corpus(n, s, 130, TFR_RT_EXAMPLE),
}
# the corpora whose clean blocks a drop-mode decoder submits without a host synchronisation once it has learned them
PIPELINED = {"cfg2", "ragged_strings", "byte_array"}


def bad_block(name, n, seed, n_bad, lencrc=False):
    sch, rt, rows, frames = CORPORA[name](n, seed)
    R_ = random.Random(seed)
    bad = sorted(R_.sample(range(n), n_bad))
    lencrc_at = min(n - 1, bad[-1] + 1 + R_.randrange(max(1, n - bad[-1] - 1))) if lencrc else None
    return sch, rt, rows, frames, corrupt(frames, sch, rows, rt, R_, bad, lencrc_at)


# ---------------------------------------------------------------------------------------------
# 1. every case and golden vector, decoded in drop mode
# ---------------------------------------------------------------------------------------------
def test_every_case(native, oracle):
    import cases as CS
    n = dropped = 0
    for c in CS.all_cases():
        sch = _schema_of_case(c)
        exp = check_fresh(native, oracle, c.data(), sch, c.record_type, getattr(c, "flags", A.TFR_F_DEFAULT) | A.TFR_F_DROP_MALFORMED,
                          getattr(c, "is_final", True), what=c.name)
        n += 1
        dropped += len(exp.dropped)
    assert n > 20 and dropped > 10, (n, dropped)


def test_golden_vectors(native, oracle):
    import test_golden as G
    dropped = 0
    for e in G.INDEX:
        sch = byte_array_schema() if e["record_type"] == 2 else G.schema_of(e)
        data = open(os.path.join(G.HERE, e["file"]), "rb").read()
        exp = check_fresh(native, oracle, data, sch, e["record_type"], e["flags"] | A.TFR_F_DROP_MALFORMED, e["is_final"], what=e["name"])
        dropped += len(exp.dropped)
    assert dropped > 5


# ---------------------------------------------------------------------------------------------
# 2. seeded corpora, a fresh decoder
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lencrc", [False, True], ids=["clean_tail", "lencrc_flip"])
@pytest.mark.parametrize("name", sorted(CORPORA))
def test_corpus_fresh_decoder(native, oracle, name, lencrc):
    n = 600 if name == "w130_general" else 1500
    for seed in (1, 2):
        sch, rt, rows, frames, data = bad_block(name, n, seed * 101 + len(name), 9, lencrc)
        exp = check_fresh(native, oracle, data, sch, rt, what=f"{name} seed {seed}")
        assert len(exp.dropped) >= 5, exp.dropped
        assert bool(exp.info["error_code"]) == lencrc, exp.info
        if lencrc:
            assert exp.info["error_code"] == A.TFR_E_CRC_LENGTH and exp.info["error_row"] > exp.info["n_rows"]


# ---------------------------------------------------------------------------------------------
# 3. a decoder in its pipelined steady state: clean, bad, clean
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CORPORA))
def test_corpus_pipelined(native, oracle, name):
    n = 600 if name == "w130_general" else 1500
    sch, rt, rows, frames, data = bad_block(name, n, 7 + len(name), 6)
    clean = b"".join(frames)
    want_clean = expected(oracle, clean, sch, rt, DROP)
    exp = expected(oracle, data, sch, rt, DROP)
    assert len(exp.dropped) >= 3
    dec = native.Decoder(sch, rt, flags=DROP)
    ff = native.Decoder(sch, rt, flags=A.TFR_F_DEFAULT)
    for _ in range(3):                                         # learning
        b = dec.submit(clean)
        check_info(b, want_clean, f"{name} learning")
        b.release()
    pipelined = name in PIPELINED

    def clean_batch(tag):
        s0 = dec.stats()
        b = dec.submit(clean)
        b.unsafe_rows_async(True)
        check_info(b, want_clean, tag)
        got = b.to_host()
        assert_columns_equal(got, want_clean.columns, None, tag)
        check_rows(b, sch, want_clean, None, tag)
        b.release()
        d = delta(s0, dec.stats())
        if pipelined:
            assert d["speculative_submits"] == 1 and d["speculative_redone"] == 0, (tag, d)
        assert d["records_dropped"] == 0, (tag, d)
        return got

    got = clean_batch(f"{name} clean before")
    bf, _ = ff.decode(clean)                                  # a clean block: bit-identical to FAILFAST
    assert_columns_equal(got, bf.to_host(), None, f"{name} clean vs FAILFAST")
    assert {k: bf.info[k] for k in want_clean.info} == want_clean.info
    bf.release()
    s0 = dec.stats()
    b = dec.submit(data)
    b.unsafe_rows_async(True)
    check_info(b, exp, f"{name} bad")
    assert_columns_equal(b.to_host(), exp.columns, None, f"{name} bad")
    check_rows(b, sch, exp, None, f"{name} bad (async)")
    b.release()
    d = delta(s0, dec.stats())
    assert d["records_dropped"] == len(exp.dropped), d
    if pipelined:
        assert d["speculative_submits"] == 1 and d["speculative_redone"] == 1, d
    clean_batch(f"{name} clean after")
    # a pipelined bad block whose rows are asked for with a partition row
    b = dec.submit(data)
    b.unsafe_rows_async(True, (P.partition_row(*PART), P.var_flags(PART[0])))
    check_info(b, exp, f"{name} bad, partitioned")
    check_rows(b, sch, exp, PART, f"{name} bad (async, partitioned)")
    b.release()
    clean_batch(f"{name} clean at the end")
    dec.close()
    ff.close()


# ---------------------------------------------------------------------------------------------
# 4. streamed in 1 MiB blocks with carry-over
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lencrc", [False, True], ids=["clean_tail", "lencrc_flip"])
@pytest.mark.parametrize("name", ["cfg2", "ragged_strings", "byte_array"])
def test_corpus_streamed(native, oracle, name, lencrc):
    n = {"cfg2": 3000, "ragged_strings": 30000, "byte_array": 20000}[name]
    sch, rt, rows, frames, data = bad_block(name, n, 31 + len(name), 40, lencrc)
    dec = native.Decoder(sch, rt, flags=DROP)
    ff = native.Decoder(sch, rt, flags=A.TFR_F_DEFAULT)
    warm = b"".join(frames)[:1 << 20]
    for d_ in (dec, ff):                                      # both in their steady state: the blocks are submitted pipelined
        for _ in range(3):
            d_.submit(warm, is_final=False).release()
    pos, blocks, dropped, stopped = 0, 0, 0, False
    while True:
        chunk = data[pos:pos + (1 << 20)]
        final = pos + len(chunk) >= len(data)
        exp = expected(oracle, chunk, sch, rt, DROP, is_final=final)
        b = dec.submit(chunk, is_final=final)
        bf = ff.submit(chunk, is_final=final)
        used = b.consumed()                                   # the frame index's count, before the block is decoded
        assert used == bf.consumed(), (blocks, used, bf.consumed())
        bf.release()
        if not exp.info["error_code"]:
            assert used == exp.info["consumed_bytes"], (blocks, used, exp.info)
        check_info(b, exp, f"{name} block {blocks}")
        assert_columns_equal(b.to_host(), exp.columns, None, f"{name} block {blocks}")
        b.release()
        dropped += len(exp.dropped)
        blocks += 1
        if exp.info["error_code"]:
            stopped = True
            break
        pos += used
        if final:
            break
    assert blocks >= 3 and dropped >= 10 and stopped == lencrc, (blocks, dropped, stopped)
    assert dec.stats()["records_dropped"] == dropped
    dec.close()
    ff.close()


# ---------------------------------------------------------------------------------------------
# 5. edge cases
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg2", "byte_array"])
def test_every_record_dropped(native, oracle, name):
    sch, rt, rows, frames = CORPORA[name](200, 5)
    data = b"".join(bytes(f[:-1]) + bytes([f[-1] ^ 0x10]) for f in frames)   # every payload CRC wrong
    exp = check_fresh(native, oracle, data, sch, rt, what=f"{name} all dropped")
    assert exp.info["n_rows"] == 0 and len(exp.dropped) == 200
    dec = native.Decoder(sch, rt, flags=DROP)
    b, _ = dec.decode(data)
    rows_, offs = b.unsafe_rows(True)
    assert len(rows_) == 0 and list(offs) == [0]
    assert all(c.n_rows == 0 for c in b.to_host())
    b.release()
    dec.close()


def test_verify_crc_off(native, oracle):
    """without TFR_F_VERIFY_CRC a payload bit flip is not a record error (unless it breaks the protobuf)"""
    sch, rt, rows, frames = cfg2_corpus(800, 9)
    R_ = random.Random(9)
    data = corrupt(frames, sch, rows, rt, R_, sorted(R_.sample(range(800), 12)))
    exp = check_fresh(native, oracle, data, sch, rt, flags=A.TFR_F_DROP_MALFORMED, what="verify off")
    with_crc = expected(oracle, data, sch, rt, DROP)
    assert len(exp.dropped) < len(with_crc.dropped)
    assert all(code != A.TFR_E_CRC_DATA for _, _, code, _ in exp.dropped)


def test_without_the_flag_nothing_is_dropped(native, oracle):
    sch, rt, rows, frames, data = bad_block("cfg2", 500, 3, 4)
    dec = native.Decoder(sch, rt)
    b, _ = dec.decode(data)
    assert b.info["error_code"] in A.RECORD_ERRORS and b.dropped() == []
    assert dec.stats()["records_dropped"] == 0
    b.release()
    dec.close()


def test_default_source_load(native, oracle, tmp_path):
    from spark_tfrecord_b200.io import DefaultSource
    sch, rt, rows, frames, data = bad_block("ragged_strings", 700, 13, 7)
    (tmp_path / "part-00000.tfrecord").write_bytes(data)
    exp = expected(oracle, data, sch, rt, DROP)
    want = [tuple(c.get(r) for c in exp.columns) for r in range(exp.info["n_rows"])]
    for mode in ("DROPMALFORMED", "dropMalformed"):
        got = DefaultSource().load(str(tmp_path), sch, {"mode": mode})
        assert got == want
    with pytest.raises(native.TfrError):
        DefaultSource().load(str(tmp_path), sch, {"mode": "FAILFAST"})
    with pytest.raises(native.TfrError):
        DefaultSource().load(str(tmp_path), sch)
    # a small block size: the block loop's carry-over and the per-block log
    from spark_tfrecord_b200.io import PartitionedFile, TFRecordFileReader
    got = list(TFRecordFileReader.readFile(None, {"mode": "DROPMALFORMED"}, PartitionedFile(str(tmp_path / "part-00000.tfrecord")), sch,
                                           block_bytes=64 << 10))
    assert got == want
