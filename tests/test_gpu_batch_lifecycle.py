"""GPU tests of a pipelined batch's lifecycle in orderings the other tests do not take: a batch released while its host copy
and its rows are still queued, or right after tfr_batch_consumed, and a redone batch whose host copy was queued before the
redo.  The lane such a batch ran on is reused afterwards, and every later batch must still be the oracle's, with no
speculative redo and no rows rebuilt (Decoder.stats())."""
import numpy as np
import pytest

from spark_tfrecord_b200 import _cabi as A
from test_gpu_decode_rows import check_batch, expected
from util import assert_columns_equal, record_offsets

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


@pytest.fixture(scope="module")
def corpus(oracle):
    """configs[1]-shaped records, the oracle's decode of them and its rows"""
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(2000, seed=41)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0
    want = oracle.decode(data, sch)
    return sch, data, want, expected(sch, want.columns, want.n_rows)


def check_columns(b, want, sch, what):
    for k in ("error_code", "error_row", "error_field", "n_rows", "consumed_bytes"):
        assert b.info[k] == want.info[k], (what, k, b.info, want.info)
    assert_columns_equal(b.to_host(), want.columns, sch.names, what)


def steady_decoder(native, oracle, corpus):
    """a decoder that has learned the corpus' shapes and row sizes: its next submits are pipelined, their rows enqueued"""
    sch, data, _, want_rows = corpus
    dec = native.Decoder(sch)
    b = dec.submit(data)
    b.unsafe_rows_async()
    check_batch(native, oracle, b, data, sch, want_rows=want_rows)
    b.release()
    return dec


def delta(s0, s1):
    return {k: s1[k] - s0[k] for k in s0}


@pytest.mark.parametrize("before_release", ["host_copy_and_rows", "consumed"])
def test_pending_batch_released_before_any_wait_frees_its_lane(native, oracle, corpus, before_release):
    sch, data, want, want_rows = corpus
    dec = steady_decoder(native, oracle, corpus)
    try:
        s0 = dec.stats()
        b = dec.submit(data)
        if before_release == "host_copy_and_rows":
            b.to_host_async()
            b.unsafe_rows_async(to_host=True)
        else:
            assert b.consumed() == len(data)
        b.release()
        more = 2 * native.Decoder.num_staging_slots()        # round robin: every lane twice, the released batch's included
        for k in range(more):
            b = dec.submit(data)
            b.to_host_async()
            b.unsafe_rows_async(to_host=True)
            check_batch(native, oracle, b, data, sch, want_rows=want_rows)
            check_columns(b, want, sch, f"submit {k} after the release ({before_release})")
            b.release()
        d = delta(s0, dec.stats())
        assert d["speculative_submits"] == more + 1 and d["speculative_redone"] == 0, d
        assert d["rows_async"] == more + (before_release == "host_copy_and_rows") and d["rows_async_rebuilt"] == 0, d
    finally:
        dec.close()


def test_host_copy_queued_before_a_redo_gives_the_redone_batch(native, oracle, corpus):
    sch, data, want, want_rows = corpus
    offs = record_offsets(np.frombuffer(data, np.uint8))
    bad = bytearray(data)
    bad[int(offs[1000]) + 40] ^= 0x10                          # a payload byte of record 1000: its data CRC fails
    want_bad = oracle.decode(bytes(bad), sch)
    assert want_bad.info["error_code"] == A.TFR_E_CRC_DATA and want_bad.info["error_row"] == 1000, want_bad.info
    dec = steady_decoder(native, oracle, corpus)
    try:
        s0 = dec.stats()
        b = dec.submit(bytes(bad))
        b.to_host_async()                                      # copies the speculative outputs that the redo replaces
        check_columns(b, want_bad, sch, "redone batch")
        b.release()
        d = delta(s0, dec.stats())
        assert d["speculative_submits"] == 1 and d["speculative_redone"] == 1, d
        b = dec.submit(data)                                   # and the decoder goes on in the steady state
        b.to_host_async()
        check_columns(b, want, sch, "the next batch")
        b.release()
        d = delta(s0, dec.stats())
        assert d["speculative_submits"] == 2 and d["speculative_redone"] == 1, d
    finally:
        dec.close()
