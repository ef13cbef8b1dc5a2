"""GPU tests of tfr_batch_rows_async: the rows of a decoded batch enqueued at submit time, with no host synchronisation once the
decoder has learned its row sizes.  Every result is compared byte for byte, offsets included, with tfr_batch_rows of the same
bytes on a fresh decoder and with oracle.unsaferow's rows of the oracle's decode (check_batch / assert_rows of
test_gpu_decode_rows).  Decoder.stats(): rows_async counts the passes enqueued without a host synchronisation,
rows_async_rebuilt those rebuilt through the synchronous path."""
import os
import subprocess
import threading

import numpy as np
import pytest

from oracle import unsaferow as U
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_decode_rows import assert_rows, check_batch, expected
from test_gpu_encode_rows import rows_of
import partition_rows as P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def fresh_rows(native, sch, data, rt=0, partition=None, is_final=True):
    """tfr_batch_rows of the same bytes on a fresh decoder (host rows, copied)"""
    dec = native.Decoder(sch, rt)
    try:
        b, _ = dec.decode(bytes(data), is_final=is_final)
        r, o = b.unsafe_rows(True, partition=partition)
        out = (r.copy(), o.copy())
        b.release()
        return out
    finally:
        dec.close()


def check_async(native, oracle, b, data, sch, rt=0, want_rows=None, partition=None, is_final=True):
    """the rows of `b` (rows enqueued asynchronously) == a fresh decoder's tfr_batch_rows == the oracle's rows"""
    fresh = fresh_rows(native, sch, data, rt, partition, is_final)
    if partition is None:
        h, _ = check_batch(native, oracle, b, data, sch, rt, is_final=is_final, want_rows=want_rows)
    else:
        h = b.unsafe_rows(True, partition=partition)
        h = (h[0].copy(), h[1].copy())
        assert_rows(sch, h, want_rows, "host rows with partition values vs oracle")
        rp, op, n, nb = b.unsafe_rows(False, partition=partition)
        assert n == len(h[1]) - 1 and nb == len(h[0])
    assert_rows(sch, h, fresh, "async rows vs a fresh decoder's tfr_batch_rows")
    return h


def delta(s0, s1):
    return {k: s1[k] - s0[k] for k in s0}


def _cfg2(n, seed):
    from oracle.corpus import cfg2_columns
    return cfg2_columns(n, seed=seed)


@pytest.mark.parametrize("to_host", [True, False])
def test_steady_state_reader_loop_from_pinned_slots(native, oracle, to_host):
    """the INTEGRATION reader loop: block k staged in slot k % 3, submitted, its rows enqueued; block k+1 submitted before
    block k's rows are read.  The first block teaches the decoder; every block submitted after that is enqueued, none rebuilt"""
    blocks = []
    for k in range(7):
        sch, cols = _cfg2(3000 + 100 * k, seed=300 + k)
        data, rc, _ = oracle.encode(cols, sch)
        wr, wo = U.cfg2_rows(cols)
        blocks.append((data, (wr, wo.astype(np.int64))))
    dec = native.Decoder(sch)
    try:
        slots = native.Decoder.num_staging_slots()
        s0 = dec.stats()

        def submit(k):
            data = blocks[k][0]
            buf = dec.staging_slot(k % slots, len(data))
            buf[:len(data)] = np.frombuffer(data, np.uint8)
            b = dec.submit((buf.ctypes.data, len(data), 0))
            b.unsafe_rows_async(to_host=to_host)
            return b

        ahead = submit(0)
        for k in range(len(blocks)):
            b, ahead = ahead, None
            assert b.consumed() == len(blocks[k][0])
            if k + 1 < len(blocks):
                ahead = submit(k + 1)
            before = dec.stats()
            check_async(native, oracle, b, blocks[k][0], sch, want_rows=blocks[k][1])
            after = dec.stats()
            assert after["rows_async_rebuilt"] == before["rows_async_rebuilt"]
            b.release()
        d = delta(s0, dec.stats())
        # block 0 teaches the decoder when its rows are built, and block 1 is submitted (its rows only recorded) before that
        assert d["rows_async"] == len(blocks) - 2, d
        assert d["rows_async_rebuilt"] == 0 and d["speculative_redone"] == 0, d
        assert d["speculative_submits"] >= len(blocks) - 2, d
    finally:
        dec.close()


@pytest.mark.parametrize("to_host", [True, False])
def test_more_blocks_in_flight_than_lanes(native, oracle, to_host):
    from oracle.corpus import cfg1_columns
    sch, cols = cfg1_columns(2000, seed=71)
    data, rc, _ = oracle.encode(cols, sch)
    want = expected(sch, oracle.decode(data, sch).columns, 2000)
    dec = native.Decoder(sch)
    try:
        b = dec.submit(data)
        b.unsafe_rows_async(to_host=to_host)                   # learning: recorded only, built by the rows call
        check_async(native, oracle, b, data, sch, want_rows=want)
        b.release()
        s0 = dec.stats()
        inflight = []
        for _ in range(5):                                     # five submitted, three lanes: a submit resolves the oldest
            b = dec.submit(data)
            b.unsafe_rows_async(to_host=to_host)
            inflight.append(b)
        for b in inflight:
            check_async(native, oracle, b, data, sch, want_rows=want)
            b.release()
        d = delta(s0, dec.stats())
        assert d["rows_async"] == 5 and d["rows_async_rebuilt"] == 0 and d["speculative_redone"] == 0, d
    finally:
        dec.close()


def test_submit_and_async_rows_return_before_the_kernels_finish(native, oracle):
    import torch
    sch, cols = _cfg2(100_000, seed=5)
    data, rc, _ = oracle.encode(cols, sch)
    dec = native.Decoder(sch)
    try:
        buf = dec.staging_slot(0, len(data))
        buf[:len(data)] = np.frombuffer(data, np.uint8)
        src = (buf.ctypes.data, len(data), 0)
        pending_seen = 0
        for it in range(4):
            b = dec.submit(src)
            b.unsafe_rows_async(to_host=True)
            busy = not torch.cuda.ExternalStream(dec.stream()).query()
            if it >= 2:                                        # learned, pools warm
                pending_seen += busy
            r, o = b.unsafe_rows(True)
            assert len(o) == 100_001
            b.release()
        assert pending_seen == 2, "the submit and the async rows call waited for the batch's kernels"
        assert dec.stats()["rows_async"] == 3
    finally:
        dec.close()


def test_partition_values(native, oracle):
    from oracle.corpus import mixed_columns
    sch, cols = mixed_columns(1500, seed=31)
    data, rc, _ = oracle.encode(cols, sch)
    want_cols = oracle.decode(data, sch).columns
    ptypes, pvals = ["string", "string", "int"], ["2024-01-02", None, -7]
    part = (P.partition_row(ptypes, pvals), P.var_flags(ptypes))
    want = P.joined_rows(sch, rows_of(want_cols, 1500), ptypes, pvals)
    dec = native.Decoder(sch)
    try:
        s0 = dec.stats()
        for it in range(4):
            b = dec.submit(data)
            b.unsafe_rows_async(to_host=it % 2 == 0, partition=part)
            check_async(native, oracle, b, data, sch, want_rows=want, partition=part)
            b.release()
        d = delta(s0, dec.stats())
        assert d["rows_async"] == 3 and d["rows_async_rebuilt"] == 0, d
    finally:
        dec.close()


def _ragged_cases(oracle):
    from oracle.corpus import cfg4_columns, mixed_columns
    rng = np.random.default_rng(17)
    sch = StructType([StructField("s", StringType()), StructField("a", ArrayType(LongType())), StructField("as", ArrayType(StringType())),
                      StructField("f", ArrayType(FloatType()))])
    rows = [("x" * int(rng.integers(0, 40)), [int(v) for v in rng.integers(-99, 99, int(rng.integers(0, 9)))],
             ["y" * int(k) for k in rng.integers(0, 7, int(rng.integers(0, 5)))], [float(v) for v in rng.random(int(rng.integers(0, 4)))])
            for _ in range(2500)]
    data, rc, _ = oracle.encode(A.columns_from_rows(sch, rows), sch)
    yield "ragged", sch, TFR_RT_EXAMPLE, data
    sch4, cols4 = cfg4_columns(800, seed=19)
    data4, rc, _ = oracle.encode(cols4, sch4, TFR_RT_SEQUENCE_EXAMPLE)
    yield "sequence_example", sch4, TFR_RT_SEQUENCE_EXAMPLE, data4
    schb = byte_array_schema()
    rowsb = [(rng.integers(0, 256, int(s), dtype=np.uint8).tobytes(),) for s in rng.integers(0, 900, 3000)]
    datab, rc, _ = oracle.encode(A.columns_from_rows(schb, rowsb, TFR_RT_BYTE_ARRAY), schb, TFR_RT_BYTE_ARRAY)
    yield "bytearray", schb, TFR_RT_BYTE_ARRAY, datab


def test_ragged_columns_sequence_example_and_bytearray(native, oracle):
    for name, sch, rt, data in _ragged_cases(oracle):
        dec = native.Decoder(sch, rt)
        try:
            s0 = dec.stats()
            for it in range(4):
                b = dec.submit(data)
                b.unsafe_rows_async(to_host=it != 2)
                check_async(native, oracle, b, data, sch, rt)
                b.release()
            d = delta(s0, dec.stats())
            assert d["rows_async"] == 3 and d["rows_async_rebuilt"] == 0, (name, d)
        finally:
            dec.close()


def _strings(oracle, lens, seed, bad=()):
    """Example records of (id: Long, s: String); the bytes are written as BinaryType so that `bad` rows can carry malformed
    UTF-8, and are read with the StringType schema"""
    rng = np.random.default_rng(seed)
    wsch = StructType([StructField("id", LongType()), StructField("s", BinaryType())])
    rows = []
    for i, l in enumerate(lens):
        v = bytes(rng.integers(97, 123, int(l), dtype=np.uint8))
        if i in bad:
            v = v[:3] + b"\xff\xfe" + v[3:]
        rows.append((i, v))
    data, rc, _ = oracle.encode(A.columns_from_rows(wsch, rows), wsch)
    assert rc == 0
    return data


STR_SCH = StructType([StructField("id", LongType()), StructField("s", StringType())])
# the same records read with 30 more (absent, so null) long columns: every row gets 240 fixed bytes the framed bytes do not have
WIDE_SCH = StructType(list(STR_SCH) + [StructField(f"n{i}", LongType()) for i in range(30)])


def _learn(native, oracle, dec, data, k=3, sch=STR_SCH):
    for _ in range(k):
        b = dec.submit(data)
        b.unsafe_rows_async()
        check_async(native, oracle, b, data, sch)
        b.release()


def _pipelined_again(native, oracle, dec, data, sch=STR_SCH):
    """the next clean batch is enqueued without a host synchronisation and not rebuilt"""
    s0 = dec.stats()
    b = dec.submit(data)
    b.unsafe_rows_async()
    check_async(native, oracle, b, data, sch)
    b.release()
    d = delta(s0, dec.stats())
    assert d["rows_async"] == 1 and d["rows_async_rebuilt"] == 0, d


def test_fallback_rows_outgrow_their_capacity(native, oracle):
    rng = np.random.default_rng(1)
    big = _strings(oracle, rng.integers(190, 211, 2000), 2)
    small = _strings(oracle, rng.integers(90, 111, 2000), 3)      # more row bytes per framed byte: the fixed part weighs more
    dec = native.Decoder(WIDE_SCH)
    try:
        _learn(native, oracle, dec, big, 4, WIDE_SCH)
        s0 = dec.stats()
        b = dec.submit(small)
        b.unsafe_rows_async()
        check_async(native, oracle, b, small, WIDE_SCH)
        b.release()
        d = delta(s0, dec.stats())
        assert d["rows_async"] == 1 and d["rows_async_rebuilt"] == 1 and d["speculative_redone"] == 0, d
        _pipelined_again(native, oracle, dec, small, WIDE_SCH)
    finally:
        dec.close()


def test_fallback_speculative_redo_after_a_payload_bit_flip(native, oracle):
    data = _strings(oracle, np.random.default_rng(4).integers(20, 60, 3000), 5)
    bad = bytearray(data)
    pos = 0
    for _ in range(1500):                                      # the payload of record 1500: its data CRC fails
        pos += 16 + int.from_bytes(data[pos:pos + 8], "little")
    bad[pos + 12 + int.from_bytes(data[pos:pos + 8], "little") // 2] ^= 0x10
    dec = native.Decoder(STR_SCH)
    try:
        _learn(native, oracle, dec, data)
        s0 = dec.stats()
        b = dec.submit(bytes(bad))
        b.unsafe_rows_async()
        h = check_async(native, oracle, b, bad, STR_SCH)
        want = oracle.decode(bytes(bad), STR_SCH)
        assert b.info["error_code"] == want.info["error_code"] != 0 and b.info["error_row"] == want.info["error_row"]
        assert len(h[1]) == want.info["n_rows"] + 1
        b.release()
        d = delta(s0, dec.stats())
        assert d["speculative_redone"] == 1 and d["rows_async"] == 1 and d["rows_async_rebuilt"] == 1, d
        _pipelined_again(native, oracle, dec, data)
    finally:
        dec.close()


def test_fallback_shape_change(native, oracle):
    sch, cols = _cfg2(3000, seed=8)
    data, rc, _ = oracle.encode(cols, sch)
    from oracle.corpus import cfg2_columns
    sch2, cols2 = cfg2_columns(3000, seed=9, float_len=5, bytes_len=16)
    data2, rc, _ = oracle.encode(cols2, sch2)
    dec = native.Decoder(sch)
    try:
        for _ in range(3):
            b = dec.submit(data)
            b.unsafe_rows_async()
            check_async(native, oracle, b, data, sch)
            b.release()
        s0 = dec.stats()
        b = dec.submit(data2)
        b.unsafe_rows_async()
        check_async(native, oracle, b, data2, sch)
        b.release()
        d = delta(s0, dec.stats())
        assert d["speculative_redone"] == 1 and d["rows_async_rebuilt"] == 1, d
        for _ in range(3):                                     # relearned: pipelined again
            s1 = dec.stats()
            b = dec.submit(data2)
            b.unsafe_rows_async()
            check_async(native, oracle, b, data2, sch)
            b.release()
        d = delta(s1, dec.stats())
        assert d["rows_async"] == 1 and d["rows_async_rebuilt"] == 0 and d["speculative_redone"] == 0, d
    finally:
        dec.close()


def test_fallback_more_records_than_provisioned(native, oracle):
    rng = np.random.default_rng(6)
    big = _strings(oracle, rng.integers(190, 211, 2000), 7)
    many = _strings(oracle, rng.integers(10, 30, 6000), 8)
    dec = native.Decoder(STR_SCH)
    try:
        _learn(native, oracle, dec, big)
        s0 = dec.stats()
        b = dec.submit(many)
        b.unsafe_rows_async()
        check_async(native, oracle, b, many, STR_SCH)
        b.release()
        d = delta(s0, dec.stats())
        assert d["speculative_redone"] == 1 and d["rows_async_rebuilt"] == 1, d
        _pipelined_again(native, oracle, dec, many)
    finally:
        dec.close()


def test_fallback_malformed_utf8_takes_the_transcoding_kernel(native, oracle):
    rng = np.random.default_rng(10)
    lens = rng.integers(5, 40, 3000)
    clean = _strings(oracle, lens, 11)
    dirty = _strings(oracle, lens, 11, bad={17, 1500})
    dec = native.Decoder(STR_SCH)
    try:
        _learn(native, oracle, dec, clean)
        s0 = dec.stats()
        b = dec.submit(dirty)
        b.unsafe_rows_async()
        check_async(native, oracle, b, dirty, STR_SCH)
        b.release()
        d = delta(s0, dec.stats())
        assert d["transcode_reruns"] == 1 and d["rows_async_rebuilt"] == 1, d
        _pipelined_again(native, oracle, dec, dirty)
    finally:
        dec.close()


def test_api_edges(native, oracle):
    # a DecimalType schema: refused at once, the columns stay readable
    dsch = StructType([StructField("x", LongType()), StructField("dec", DecimalType())])
    ddata, rc, _ = oracle.encode(A.columns_from_rows(dsch, [(1, 1.5), (2, 2.5)]), dsch)
    dec = native.Decoder(dsch)
    try:
        b = dec.submit(ddata)
        with pytest.raises(native.TfrError) as ei:
            b.unsafe_rows_async()
        assert ei.value.code == A.TFR_E_UNSUPPORTED_TYPE and "dec" in str(ei.value)
        assert b.to_host()[0].n_rows == 2
        b.release()
    finally:
        dec.close()
    data = _strings(oracle, np.random.default_rng(12).integers(0, 50, 1000), 13)
    want = oracle.decode(data, STR_SCH)
    p1 = (P.partition_row(["int"], [5]), P.var_flags(["int"]))
    p2 = (P.partition_row(["int"], [6]), P.var_flags(["int"]))
    want1 = P.joined_rows(STR_SCH, rows_of(want.columns, 1000), ["int"], [5])
    dec = native.Decoder(STR_SCH)
    try:
        _learn(native, oracle, dec, data, 2)
        # repeated async calls, then a read with another partition row: refused, the rows asked for stay intact
        b = dec.submit(data)
        s0 = dec.stats()
        b.unsafe_rows_async(to_host=False, partition=p1)
        b.unsafe_rows_async(to_host=False, partition=p1)
        b.unsafe_rows_async(to_host=True, partition=p1)        # adds only the copy
        with pytest.raises(native.TfrError) as ei:
            b.unsafe_rows_async(partition=p2)
        assert ei.value.code == A.TFR_E_INVALID_ARG
        with pytest.raises(native.TfrError) as ei:
            b.unsafe_rows(True, partition=p2)
        assert ei.value.code == A.TFR_E_INVALID_ARG
        with pytest.raises(native.TfrError) as ei:
            b.unsafe_rows(True)
        assert ei.value.code == A.TFR_E_INVALID_ARG
        check_async(native, oracle, b, data, STR_SCH, want_rows=want1, partition=p1)
        b.unsafe_rows_async(partition=p1)                      # after the rows were read: nothing
        assert delta(s0, dec.stats())["rows_async"] == 1
        b.release()
        # batches released with rows enqueued and never read
        for _ in range(5):
            b = dec.submit(data)
            b.unsafe_rows_async(to_host=True)
            b.release()
        _pipelined_again(native, oracle, dec, data)
        # a decoder destroyed with batches in flight, rows enqueued
        held = []
        for _ in range(3):
            b = dec.submit(data)
            b.unsafe_rows_async()
            held.append(b)
    finally:
        dec.close()
    r, o = held[0].unsafe_rows(True)                           # the batches keep the decoder alive
    assert_rows(STR_SCH, (r.copy(), o.copy()), fresh_rows(native, STR_SCH, data), "rows of a batch that outlived its decoder")
    for b in held:
        b.release()


def test_four_reader_threads_each_with_its_own_decoder(native, oracle):
    inputs = []
    for t in range(4):
        sch, cols = _cfg2(2500, seed=60 + t)
        data, rc, _ = oracle.encode(cols, sch)
        wr, wo = U.cfg2_rows(cols)
        inputs.append((sch, data, (wr, wo.astype(np.int64))))
    errors = []

    def reader(t):
        try:
            sch, data, want = inputs[t]
            dec = native.Decoder(sch)
            try:
                ahead = dec.submit(data)
                ahead.unsafe_rows_async(to_host=t % 2 == 0)
                for k in range(6):
                    b, ahead = ahead, None
                    if k < 5:
                        ahead = dec.submit(data)
                        ahead.unsafe_rows_async(to_host=t % 2 == 0)
                    r, o = b.unsafe_rows(True)
                    assert_rows(sch, (r, o), want, f"thread {t} block {k}")
                    b.release()
                st = dec.stats()                               # (blocks 0 and 1 asked for rows before the decoder learned)
                assert st["rows_async"] == 4 and st["rows_async_rebuilt"] == 0, st
            finally:
                dec.close()
        except BaseException as e:          # noqa: BLE001 -- reported by the main thread
            errors.append((t, e))

    threads = [threading.Thread(target=reader, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors


# ---- the C emulator of the row-reading BlockIterator (tests/emulator/rowread_emulator.c) ----
def _fnv(b: bytes) -> int:
    h = 0xcbf29ce484222325
    for x in b:
        h = ((h ^ x) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def _oracle_row_sums(oracle, sch, data):
    want = oracle.decode(np.frombuffer(data, np.uint8), sch)
    n = want.info["n_rows"]
    rows, offs = U.unsafe_rows(sch, rows_of(want.columns, n))
    return ["%016x" % _fnv(bytes(rows[offs[i]:offs[i + 1]])) for i in range(n)], want.info


@pytest.fixture(scope="module")
def rowread_file(native, oracle, tmp_path_factory):
    from test_encode_pipeline_host import build_emulator, emulator_schema
    from test_rows_async_host import build_rowread
    d = tmp_path_factory.mktemp("rowread")
    writer = build_emulator(str(d / "rowwrite"))
    reader = build_rowread(str(d / "rowread"))
    n = 30000
    p = subprocess.run([writer, "rowwrite", str(d), str(n), "4000"], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    path = os.path.join(str(d), "part-00000.tfrecord")
    return reader, path, emulator_schema(), n


def _run_rowread(reader, path, block):
    p = subprocess.run([reader, "rowread", path, str(block)], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr
    lines = p.stdout.splitlines()
    st = [l for l in lines if l.startswith("status ")]
    assert len(st) == 1, lines[-3:]
    sums = [l for l in lines if len(l) == 16 and not l.startswith(("status", "rowread"))]
    f = st[0].split()
    return sums, int(f[1]), int(f[3]), lines[-1]


@pytest.mark.parametrize("block", [4096, 1 << 20, 64 << 20])
def test_emulated_rowread_of_a_rowwrite_file(oracle, rowread_file, block):
    reader, path, sch, n = rowread_file
    data = open(path, "rb").read()
    want, info = _oracle_row_sums(oracle, sch, data)
    assert info["error_code"] == 0 and len(want) == n
    sums, code, err_row, stats = _run_rowread(reader, path, block)
    assert code == 0 and err_row == -1, stats
    assert sums == want, f"block {block}: first differing row {next(i for i, (a, b) in enumerate(zip(sums, want)) if a != b) if len(sums) == len(want) else len(sums)}"
    if block == 1 << 20:
        assert "rows_rebuilt=0" in stats and "rows_async=0" not in stats, stats


def test_emulated_rowread_stops_at_a_corrupt_record(oracle, rowread_file, tmp_path):
    reader, path, sch, n = rowread_file
    data = bytearray(open(path, "rb").read())
    data[len(data) // 2] ^= 0x04                               # a payload byte of a record mid-file: its data CRC fails
    bad = str(tmp_path / "bad.tfrecord")
    open(bad, "wb").write(bytes(data))
    want, info = _oracle_row_sums(oracle, sch, bytes(data))
    assert info["error_code"] != 0
    for block in (4096, 1 << 20):
        sums, code, err_row, stats = _run_rowread(reader, bad, block)
        assert code == info["error_code"], (code, info)
        assert sums == want[:len(sums)] and len(sums) == len(want), (block, len(sums), len(want))
