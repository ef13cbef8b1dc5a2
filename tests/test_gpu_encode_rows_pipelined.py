"""GPU tests of the pipelined UnsafeRow encode (tfr_encode_rows_submit / tfr_encoded_*): a Spark writer task keeps up to
tfr_encoder_num_row_slots() flushes in flight.  Every result is compared byte for byte with tfr_encode_rows of the same rows on
a separate encoder and with the oracle writer, every error with tfr_encode_rows' status and row, and the concatenated output
is decoded back with CRC checks on.  The stats show which path each flush took: the speculative one (sized from what the
encoder learned, no host synchronisation) or a redo through the synchronous path after the device raised a flag."""
import os
import subprocess
import threading

import numpy as np
import pytest

from oracle import unsaferow as U
from oracle.corpus import cfg2_columns, cfg4_columns
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


class Flush:
    """one flush: its rows (uint8, int32 offsets), and what tfr_encode_rows makes of them (bytes, or (code, row))"""

    def __init__(self, native, sch, rt, data, offs, cols=None, oracle=None):
        self.sch, self.rt, self.data, self.offs = sch, rt, data, offs
        ref = native.Encoder(sch, rt)
        try:
            ref.encode_rows(data, offs)
            self.want, self.err = ref.result_host(), None
        except native.TfrError as e:
            self.want, self.err = None, (e.code, e.row)
        finally:
            ref.close()
        if cols is not None and oracle is not None:
            w, rc, _ = oracle.encode(cols, sch, rt)
            assert rc == 0 and w == self.want, "tfr_encode_rows differs from the oracle writer"


def cfg2_flush(native, oracle, n, seed, small_ints=False, bytes_len=16, negate=False):
    sch, cols = cfg2_columns(n, seed=seed, small_ints=small_ints, bytes_len=bytes_len)
    if negate:
        for c in cols[:32]:
            c.values[:] = -c.values - 1
    data, offs = U.cfg2_rows(cols, bytes_len=bytes_len)
    return Flush(native, sch, 0, data, offs, cols, oracle)


def rows_flush(native, oracle, sch, rows, rt=0):
    data, offs = U.unsafe_rows(sch, rows)
    return Flush(native, sch, rt, data, offs, A.columns_from_rows(sch, rows, rt), oracle)


def check_result(native, f, s):
    if f.err is None:
        s.wait()
        got = s.result_host()
        assert got == f.want, f"len {len(got)} vs {len(f.want)}"
        return got
    with pytest.raises(native.TfrError) as ei:
        s.wait()
    assert (ei.value.code, ei.value.row) == f.err
    return b""


def decode_back(native, sch, rt, blob, n_rows):
    dec = native.Decoder(sch, rt)
    try:
        b, used = dec.decode(blob)
        assert b.info["error_code"] == 0 and used == len(blob) and b.n_rows == n_rows, b.info
        b.release()
    finally:
        dec.close()


def writer_loop(native, enc, flushes, use_slots=True):
    """the RowWriter loop of INTEGRATION.md: flush k goes through slot k % S; before a slot is refilled, the submission that
    read it is waited on and its bytes written out; close() drains in order"""
    S = native.Encoder.num_row_slots()
    pending = [None] * S
    out = []

    def drain(k):
        f, s = pending[k]
        out.append(check_result(native, f, s))
        s.release()
        pending[k] = None

    for i, f in enumerate(flushes):
        k = i % S
        if pending[k] is not None:
            drain(k)
        if use_slots:
            st = enc.row_staging_slot(k, len(f.data))
            st[:len(f.data)] = f.data
            s = enc.submit_rows((st.ctypes.data, len(f.data), 0), f.offs)
        else:
            s = enc.submit_rows(f.data, f.offs)
        pending[k] = (f, s)
    for j in range(len(flushes), len(flushes) + S):
        if pending[j % S] is not None:
            drain(j % S)
    return b"".join(out)


# ---- 1. parity in steady state --------------------------------------------------------------------------------------
def test_steady_state_example(native, oracle):
    flushes = [cfg2_flush(native, oracle, 3000 + 17 * i, seed=100 + i) for i in range(9)]
    enc = native.Encoder(flushes[0].sch)
    try:
        blob = writer_loop(native, enc, flushes)
        st = enc.stats()
    finally:
        enc.close()
    assert blob == b"".join(f.want for f in flushes)
    assert st["submits"] == 9 and st["speculative_submits"] >= 9 - 2 and st["speculative_redone"] == 0, st
    decode_back(native, flushes[0].sch, 0, blob, sum(len(f.offs) - 1 for f in flushes))


def test_steady_state_sequence_example_general_emit(native, oracle):
    flushes = []
    for i in range(8):
        sch, cols = cfg4_columns(400, seed=300 + i)
        flushes.append(Flush(native, sch, TFR_RT_SEQUENCE_EXAMPLE, *_rows_of_cols(sch, cols), cols, oracle))
    enc = native.Encoder(flushes[0].sch, TFR_RT_SEQUENCE_EXAMPLE)
    try:
        blob = writer_loop(native, enc, flushes, use_slots=False)
        st = enc.stats()
    finally:
        enc.close()
    assert blob == b"".join(f.want for f in flushes)
    assert st["speculative_submits"] >= 8 - 2 and st["speculative_redone"] == 0 and st["general_emit"] > 0, st
    decode_back(native, flushes[0].sch, TFR_RT_SEQUENCE_EXAMPLE, blob, 8 * 400)


def _rows_of_cols(sch, cols):
    n = cols[0].n_rows
    rows = []
    for r in range(n):
        row = []
        for c in cols:
            if c.depth == 0:
                row.append(c.values[r])
            else:
                o0, o1 = c.offsets[0], c.offsets[1]
                row.append([list(c.values[o1[s]:o1[s + 1]]) for s in range(o0[r], o0[r + 1])])
        rows.append(tuple(row))
    return U.unsafe_rows(sch, rows)


def _bytearray_flush(native, oracle, seed, n=2000, lo=100, hi=200, long_row=None):
    rng = np.random.default_rng(seed)
    rows = [(rng.integers(0, 256, int(k), dtype=np.uint8).tobytes(),) for k in rng.integers(lo, hi, n)]
    if long_row is not None:
        rows[long_row[0]] = (rng.integers(0, 256, long_row[1], dtype=np.uint8).tobytes(),)
    return rows_flush(native, oracle, byte_array_schema(), rows, TFR_RT_BYTE_ARRAY)


def test_steady_state_bytearray(native, oracle):
    flushes = [_bytearray_flush(native, oracle, 40 + i) for i in range(8)]
    enc = native.Encoder(flushes[0].sch, TFR_RT_BYTE_ARRAY)
    try:
        blob = writer_loop(native, enc, flushes)
        st = enc.stats()
    finally:
        enc.close()
    assert blob == b"".join(f.want for f in flushes)
    assert st["speculative_submits"] >= 8 - 2 and st["speculative_redone"] == 0, st
    decode_back(native, flushes[0].sch, TFR_RT_BYTE_ARRAY, blob, 8 * 2000)


# ---- 2. submit does not block ----------------------------------------------------------------------------------------
def test_submit_returns_while_the_kernel_stream_is_busy(native, oracle):
    import torch
    flushes = [cfg2_flush(native, oracle, 4000, seed=500 + i) for i in range(4)]
    enc = native.Encoder(flushes[0].sch)
    try:
        S = native.Encoder.num_row_slots()
        slots = [enc.row_staging_slot(k, len(flushes[0].data) + 4096) for k in range(S)]
        slots[0][:len(flushes[0].data)] = flushes[0].data
        s = enc.submit_rows((slots[0].ctypes.data, len(flushes[0].data), 0), flushes[0].offs)   # learns
        check_result(native, flushes[0], s)
        s.release()
        for k in range(S):
            slots[k][:len(flushes[k + 1].data)] = flushes[k + 1].data
        stream = torch.cuda.ExternalStream(enc.stream())
        before = enc.stats()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(400_000_000)          # a fixed-length busy kernel of about 0.2 s at 1.98 GHz
        subs = [enc.submit_rows((slots[k].ctypes.data, len(flushes[k + 1].data), 0), flushes[k + 1].offs) for k in range(S)]
        assert not stream.query(), "a submit waited for the kernel stream"
        after = enc.stats()
        assert after["speculative_submits"] - before["speculative_submits"] == S, (before, after)
        for k, s in enumerate(subs):
            check_result(native, flushes[k + 1], s)
            s.release()
        assert enc.stats()["speculative_redone"] == 0
    finally:
        enc.close()


# ---- 3. every redo path, once each -----------------------------------------------------------------------------------
def _err_schema():
    return StructType([StructField("a", LongType(), nullable=False), StructField("s", StringType()), StructField("v", ArrayType(LongType()))])


def _err_rows(n, seed, null_at=None):
    return [(None if i == null_at else i * seed, "s" * ((i + seed) % 9), list(range((i + seed) % 5))) for i in range(n)]


def _malform(f, r):
    """slot of field s in row r points past the row: TFR_E_INVALID_ARG at row r"""
    data = f.data.copy()
    p = int(f.offs[r]) + 8 + 8 * 1
    data[p:p + 8] = np.frombuffer(((1 << 40) | 3).to_bytes(8, "little"), np.uint8)
    return data


def _redo_case(native, oracle, learn, bad, after):
    """learn on `learn` (flushes, waited one by one), then `bad` must be redone exactly once with the synchronous
    result, and `after` goes back to the speculative path"""
    enc = native.Encoder(learn[0].sch, learn[0].rt)
    try:
        for f in learn:
            s = enc.submit_rows(f.data, f.offs)
            check_result(native, f, s)
            s.release()
        st0 = enc.stats()
        assert st0["speculative_submits"] >= len(learn) - 1, st0
        s = enc.submit_rows(bad.data, bad.offs)
        check_result(native, bad, s)
        s.release()
        st1 = enc.stats()
        assert st1["speculative_submits"] == st0["speculative_submits"] + 1, (st0, st1)
        assert st1["speculative_redone"] == st0["speculative_redone"] + 1, (st0, st1)
        s = enc.submit_rows(after.data, after.offs)
        check_result(native, after, s)
        s.release()
        st2 = enc.stats()
        assert st2["speculative_submits"] == st1["speculative_submits"] + 1 and st2["speculative_redone"] == st1["speculative_redone"], (st1, st2)
    finally:
        enc.close()


def test_redo_records_outgrow_the_tile_slot(native, oracle):
    sch = _err_schema()
    learn = [rows_flush(native, oracle, sch, _err_rows(3000, 3 + i)) for i in range(2)]
    rows = _err_rows(3000, 9)
    rows[1500] = (rows[1500][0], "L" * 3000, rows[1500][2])        # one record 30x the others: past the learned tile slot
    _redo_case(native, oracle, learn, rows_flush(native, oracle, sch, rows), rows_flush(native, oracle, sch, _err_rows(3000, 11)))


def test_redo_output_per_input_byte_jumps(native, oracle):
    learn = [cfg2_flush(native, oracle, 3000, seed=620 + i, small_ints=True) for i in range(2)]
    bad = cfg2_flush(native, oracle, 3000, seed=630, small_ints=True, negate=True)
    assert len(bad.want) > 1.1 * len(learn[0].want)
    _redo_case(native, oracle, learn, bad, cfg2_flush(native, oracle, 3000, seed=631, small_ints=True))


def test_redo_bytearray_longer_payload(native, oracle):
    learn = [_bytearray_flush(native, oracle, 700 + i) for i in range(2)]
    _redo_case(native, oracle, learn, _bytearray_flush(native, oracle, 710, long_row=(1234, 5000)), _bytearray_flush(native, oracle, 711))


def test_redo_null_in_nonnullable(native, oracle):
    sch = _err_schema()
    learn = [rows_flush(native, oracle, sch, _err_rows(3000, 3 + i)) for i in range(2)]
    data, offs = U.unsafe_rows(sch, _err_rows(3000, 9, null_at=1777))
    bad = Flush(native, sch, 0, data, offs)
    assert bad.err == (A.TFR_E_NULL_IN_NONNULL, 1777)
    _redo_case(native, oracle, learn, bad, rows_flush(native, oracle, sch, _err_rows(3000, 11)))


def test_redo_malformed_row(native, oracle):
    sch = _err_schema()
    learn = [rows_flush(native, oracle, sch, _err_rows(3000, 3 + i)) for i in range(2)]
    good = rows_flush(native, oracle, sch, _err_rows(3000, 9))
    bad = Flush(native, sch, 0, _malform(good, 2100), good.offs)
    assert bad.err == (A.TFR_E_INVALID_ARG, 2100)
    _redo_case(native, oracle, learn, bad, rows_flush(native, oracle, sch, _err_rows(3000, 11)))


def test_redo_malformed_before_null(native, oracle):
    sch = _err_schema()
    learn = [rows_flush(native, oracle, sch, _err_rows(3000, 3 + i)) for i in range(2)]
    data, offs = U.unsafe_rows(sch, _err_rows(3000, 9, null_at=2500))
    nul = Flush(native, sch, 0, data, offs)
    bad = Flush(native, sch, 0, _malform(nul, 1200), offs)
    assert bad.err == (A.TFR_E_INVALID_ARG, 1200)
    _redo_case(native, oracle, learn, bad, rows_flush(native, oracle, sch, _err_rows(3000, 11)))


def test_topup_when_the_batch_is_a_little_larger_than_predicted(native, oracle):
    sch, cols = cfg2_columns(3000, seed=800, small_ints=True)
    data, offs = U.cfg2_rows(cols)
    first = Flush(native, sch, 0, data, offs, cols, oracle)
    for r in range(0, 3000, 100):                    # 30 small ints of 1 varint byte become 2 bytes: 30 more bytes out
        cols[0].values[r] = 300
    data2, offs2 = U.cfg2_rows(cols)
    grown = Flush(native, sch, 0, data2, offs2, cols, oracle)
    assert len(grown.want) == len(first.want) + 30
    enc = native.Encoder(sch)
    try:
        for f in (first, first, grown):
            s = enc.submit_rows(f.data, f.offs)
            check_result(native, f, s)
            s.release()
        st = enc.stats()
    finally:
        enc.close()
    assert st["speculative_submits"] == 2 and st["speculative_redone"] == 0 and st["host_topups"] == 1, st


# ---- 4. lifetime -----------------------------------------------------------------------------------------------------
def test_release_without_wait_then_keep_submitting(native, oracle):
    flushes = [cfg2_flush(native, oracle, 2000, seed=900 + i) for i in range(6)]
    enc = native.Encoder(flushes[0].sch)
    try:
        s = enc.submit_rows(flushes[0].data, flushes[0].offs)
        check_result(native, flushes[0], s)
        s.release()
        enc.submit_rows(flushes[1].data, flushes[1].offs).release()        # nobody waits for it
        enc.submit_rows(flushes[2].data, flushes[2].offs).release()
        blob = writer_loop(native, enc, flushes[3:])
        assert blob == b"".join(f.want for f in flushes[3:])
    finally:
        enc.close()


def test_more_submissions_than_slots_without_waiting(native, oracle):
    S = 3
    flushes = [cfg2_flush(native, oracle, 2000, seed=950 + i) for i in range(S + 2)]
    enc = native.Encoder(flushes[0].sch)
    try:
        assert native.Encoder.num_row_slots() == S
        subs = [enc.submit_rows(f.data, f.offs) for f in flushes]     # the oldest are waited for implicitly
        for f, s in zip(flushes, subs):
            check_result(native, f, s)
            assert s.result_device()[1] == len(f.want)
        for s in subs:
            s.release()
    finally:
        enc.close()


def test_synchronous_calls_between_submissions(native, oracle):
    flushes = [cfg2_flush(native, oracle, 2000, seed=1000 + i) for i in range(4)]
    sch, cols = cfg2_columns(700, seed=1010)
    want_cols, rc, _ = oracle.encode(cols, sch)
    assert rc == 0
    enc = native.Encoder(flushes[0].sch)
    try:
        s0 = enc.submit_rows(flushes[0].data, flushes[0].offs)
        s1 = enc.submit_rows(flushes[1].data, flushes[1].offs)
        enc.encode_rows(flushes[2].data, flushes[2].offs)
        assert enc.result_host() == flushes[2].want
        s2 = enc.submit_rows(flushes[3].data, flushes[3].offs)
        assert enc.encode(cols) == want_cols
        for f, s in zip((flushes[0], flushes[1], flushes[3]), (s0, s1, s2)):
            check_result(native, f, s)
        assert enc.result_host() == want_cols, "result_host is the last synchronous call's result"
        for s in (s0, s1, s2):
            s.release()
    finally:
        enc.close()


def test_refill_a_slot_after_its_wait(native, oracle):
    flushes = [cfg2_flush(native, oracle, 2500, seed=1100 + i) for i in range(3)]
    enc = native.Encoder(flushes[0].sch)
    try:
        held = []
        for f in flushes:
            st = enc.row_staging_slot(0, len(f.data))
            st[:len(f.data)] = f.data
            s = enc.submit_rows((st.ctypes.data, len(f.data), 0), f.offs)
            check_result(native, f, s)
            held.append(s)                          # kept: its bytes must survive the slot's reuse
        for f, s in zip(flushes, held):
            assert s.result_host() == f.want
            s.release()
    finally:
        enc.close()


def test_close_with_submissions_in_flight(native, oracle):
    flushes = [cfg2_flush(native, oracle, 2000, seed=1200 + i) for i in range(4)]
    enc = native.Encoder(flushes[0].sch)
    s = enc.submit_rows(flushes[0].data, flushes[0].offs)
    check_result(native, flushes[0], s)
    subs = [enc.submit_rows(f.data, f.offs) for f in flushes[1:]]
    enc.close()
    for x in subs + [s]:
        x.release()                                 # (the encoder has freed them)


def test_zero_row_submissions(native, oracle):
    flushes = [cfg2_flush(native, oracle, 2000, seed=1300 + i) for i in range(2)]
    enc = native.Encoder(flushes[0].sch)
    try:
        z = enc.submit_rows(np.zeros(0, np.uint8), np.zeros(1, np.int32))
        assert z.result_host() == b"" and z.result_device()[1] == 0
        z.release()
        out = []
        for f in flushes:
            s = enc.submit_rows(f.data, f.offs)
            z = enc.submit_rows(np.zeros(0, np.uint8), np.zeros(1, np.int32))
            out.append(check_result(native, f, s))
            z.wait()
            z.release()
            s.release()
        assert b"".join(out) == b"".join(f.want for f in flushes)
    finally:
        enc.close()


# ---- 5. concurrency --------------------------------------------------------------------------------------------------
def test_task_threads_each_with_a_pipelined_writer(native, oracle):
    work = {t: [cfg2_flush(native, oracle, 1500 + 100 * t, seed=2000 + 10 * t + i) for i in range(6)] for t in range(4)}
    errors, files = [], {}

    def task(t):
        try:
            enc = native.Encoder(work[t][0].sch)
            try:
                files[t] = writer_loop(native, enc, work[t])
            finally:
                enc.close()
        except BaseException as e:        # noqa: BLE001 -- reported below
            errors.append((t, repr(e)))

    threads = [threading.Thread(target=task, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in range(4):
        assert files[t] == b"".join(f.want for f in work[t]), f"task {t}"


# ---- 6. the C emulator's pipelined RowWriter -------------------------------------------------------------------------
def test_emulator_rowwrite_file_reads_back_as_the_generated_rows(native, oracle, tmp_path):
    from test_encode_pipeline_host import build_emulator, emulator_schema, emulator_rows
    exe = build_emulator(str(tmp_path / "emu"))
    n = 5000
    p = subprocess.run([exe, "rowwrite", str(tmp_path), str(n), "700"], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    path = os.path.join(str(tmp_path), "part-00000.tfrecord")
    data = open(path, "rb").read()
    sch = emulator_schema()
    got = oracle.decode(np.frombuffer(data, np.uint8), sch)
    assert got.info["error_code"] == 0 and got.n_rows == n
    assert "rowwrite ok" in p.stdout and "redone=0" in p.stdout, p.stdout
    want = A.columns_from_rows(sch, emulator_rows(n))
    from util import assert_columns_equal
    assert_columns_equal(got.columns, want, sch.names, "emulator rowwrite")
