"""GPU tests of a decoded batch's column views, read three ways: the device columns (tfr_batch_columns, copied out through
torch), the host copy (tfr_batch_to_host, with and without a tfr_batch_to_host_async enqueued right after the submit) and
the Arrow C Data Interface export (Batch.to_arrow).  Every reader must give the oracle's columns, for every kind of batch
the decoder builds its outputs for: the synchronous general path, the tile kernel in count mode and in uniform mode,
pipelined ragged and uniform batches, a redone pipelined batch, ByteArray rows, an empty block and a block holding only
a partial record, DROPMALFORMED with drops, PERMISSIVE with and without a corrupt-record column and with every record bad,
and a TFR_F_RESYNC batch with lost regions.  A batch without rows also has its views pinned pointer by pointer: every
offsets level of a variable-width column points at its one zero entry in the fixed block, and its values are null."""
import struct

import numpy as np
import pytest

import test_gpu_drop_malformed as D
import test_gpu_permissive as PM
import test_gpu_resync as RS
from oracle import corpus
from spark_tfrecord_b200._cabi import _LEAF_DTYPE, HostColumn
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_decode_rows import _Dev
from util import assert_columns_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


# ---------------------------------------------------------------------------------------------
# the three readers
# ---------------------------------------------------------------------------------------------
def _dev_array(ptr, n, dt):
    import torch
    if not ptr or n == 0:
        return np.zeros(0, dt)
    nb = n * np.dtype(dt).itemsize
    return torch.as_tensor(_Dev(ptr, nb, "|u1"), device="cuda").cpu().numpy().view(dt)


def device_columns(b):
    out = []
    for c in b.device_columns():
        offsets = [_dev_array(c.offsets[l], c.n_offsets[l], np.int32) for l in range(c.n_levels)]
        out.append(HostColumn(c.elem_type, c.depth, c.n_rows, _dev_array(c.validity, (c.n_rows + 7) // 8, np.uint8), offsets,
                              _dev_array(c.values, c.n_values, _LEAF_DTYPE[c.elem_type]), null_count=c.null_count))
    return out


def _same(g, w):
    if isinstance(w, float):
        return isinstance(g, float) and struct.pack("<d", g) == struct.pack("<d", w)
    if isinstance(w, list):
        return isinstance(g, list) and len(g) == len(w) and all(_same(x, y) for x, y in zip(g, w))
    return g == w


def check_arrow(arrs, want, what):
    assert len(arrs) == len(want), what
    for i, (arr, col) in enumerate(zip(arrs, want)):
        arr.validate(full=True)
        assert len(arr) == col.n_rows and arr.null_count == col.null_count, f"{what} arrow col {i}"
        for r, g in enumerate(arr.to_pylist()):
            assert _same(g, col.get(r)), f"{what} arrow col {i} row {r}: {g!r} != {col.get(r)!r}"


def check_readers(b, want, what):
    assert b.n_rows == (want[0].n_rows if want else 0), what
    assert_columns_equal(device_columns(b), want, None, f"{what} device")
    assert_columns_equal(b.to_host(), want, None, f"{what} to_host")
    check_arrow(b.to_arrow(), want, what)


def check_empty_views(b, sch, rt, what):
    """a batch without rows: level 0 of a variable-width column is one zero entry, every deeper level aliases it, and the
    column has no values buffer"""
    for f, c in enumerate(b.device_columns()):
        assert c.n_rows == 0 and c.validity, f"{what} col {f}"
        if c.n_levels == 0:
            assert c.values or c.elem_type == TFR_T_NULL, f"{what} col {f}"
            continue
        assert not c.values and c.n_values == 0, f"{what} col {f}: values of an empty variable-width column"
        for l in range(c.n_levels):
            assert c.offsets[l] == c.offsets[0] and c.n_offsets[l] == 1, f"{what} col {f} level {l}"


# ---------------------------------------------------------------------------------------------
# the batch kinds: each run yields (tag, batch, oracle columns); `early` enqueues the host copy right after the submit
# ---------------------------------------------------------------------------------------------
def _submit(dec, data, early, is_final=True):
    b = dec.submit(data, is_final=is_final)
    if early:
        b.to_host_async()
    return b


def _uniform_corpus(n, seed):
    """configs[1] without its binary columns: every variable-width column has the same count in every row"""
    sch, cols = corpus.cfg2_columns(n, seed=seed, n_bytes=0)
    rows = [tuple(c.get(r) for c in cols) for r in range(n)]
    import wire_rewrite as W
    from oracle import pyref
    return sch, TFR_RT_EXAMPLE, rows, [pyref.frame_fast(W.canonical(sch, row)) for row in rows]


CORPORA = dict(D.CORPORA, uniform=_uniform_corpus)


def _stat_delta(dec, s0, **want):
    d = D.delta(s0, dec.stats())
    assert all(d[k] == v for k, v in want.items()), (want, d)


def run_fresh(name, n, stat):
    """the first batch of a fresh decoder, which takes the synchronous path"""
    def run(native, oracle, early):
        sch, rt, rows, frames = CORPORA[name](n, 3)
        data = b"".join(frames)
        dec = native.Decoder(sch, rt)
        s0 = dec.stats()
        yield "first batch", _submit(dec, data, early), oracle.decode(data, sch, rt).columns
        _stat_delta(dec, s0, **{stat: 1, "speculative_submits": 0})
        dec.close()
    return run


def run_tile_uniform(native, oracle, early):
    """shapes learned, then a block too small to pipeline: the synchronous tile kernel writes every column in one pass"""
    sch, rt, rows, frames = CORPORA["uniform"](400, 4)
    dec = native.Decoder(sch, rt)
    dec.submit(b"".join(frames)).release()
    k = max(1, max(i for i in range(1, len(frames)) if sum(map(len, frames[:i])) < 4096))
    small = b"".join(frames[:k])
    s0 = dec.stats()
    yield f"{k} records", _submit(dec, small, early), oracle.decode(small, sch, rt).columns
    _stat_delta(dec, s0, batches=1, count_mode_batches=0, general_path_batches=0, speculative_submits=0)
    dec.close()


def run_pipelined(name, n):
    """a decoder in its steady state: the batch is submitted without a host synchronisation and resolved clean"""
    def run(native, oracle, early):
        sch, rt, rows, frames = CORPORA[name](n, 5)
        data = b"".join(frames)
        want = oracle.decode(data, sch, rt).columns
        dec = native.Decoder(sch, rt)
        for _ in range(3):
            dec.submit(data).release()
        for k in range(2):
            s0 = dec.stats()
            yield f"pipelined {k}", _submit(dec, data, early), want
            _stat_delta(dec, s0, speculative_submits=1, speculative_redone=0)
        dec.close()
    return run


def run_bytes(native, oracle, early):
    sch, rt, rows, frames = CORPORA["byte_array"](1500, 6)
    data = b"".join(frames)
    want = oracle.decode(data, sch, rt).columns
    dec = native.Decoder(sch, rt)
    s0 = dec.stats()
    yield "synchronous", _submit(dec, data, early), want
    _stat_delta(dec, s0, count_mode_batches=1, speculative_submits=0)
    dec.submit(data).release()
    s0 = dec.stats()
    yield "pipelined", _submit(dec, data, early), want
    _stat_delta(dec, s0, speculative_submits=1, speculative_redone=0)
    dec.close()


def run_redone(native, oracle, early):
    """a pipelined drop-mode batch whose verdict sends it through the synchronous path again"""
    sch, rt, rows, frames, data = D.bad_block("cfg2", 1500, 8, 6)
    clean = b"".join(frames)
    dec = native.Decoder(sch, rt, flags=D.DROP)
    for _ in range(3):
        dec.submit(clean).release()
    s0 = dec.stats()
    yield "redone", _submit(dec, data, early), D.expected(oracle, data, sch, rt, D.DROP).columns
    _stat_delta(dec, s0, speculative_submits=1, speculative_redone=1)
    dec.close()


def run_empty(native, oracle, early):
    for name in ("cfg2", "sequence_example", "byte_array"):
        sch, rt, rows, frames = CORPORA[name](20, 7)
        for tag, data, final in (("empty block", b"", True), ("partial record", frames[0][:len(frames[0]) // 2], False)):
            dec = native.Decoder(sch, rt)
            b = _submit(dec, data, early, is_final=final)
            want = oracle.decode(data, sch, rt, is_final=final)
            assert want.info["n_rows"] == 0 and not want.info["error_code"] and b.info["error_code"] == 0
            check_empty_views(b, sch, rt, f"{name} {tag}")
            yield f"{name} {tag}", b, want.columns
            dec.close()


def run_drop(native, oracle, early):
    for name in ("cfg2", "sequence_example"):
        sch, rt, rows, frames, data = D.bad_block(name, 1500, 9, 9)
        exp = D.expected(oracle, data, sch, rt, D.DROP)
        assert len(exp.dropped) >= 5
        dec = native.Decoder(sch, rt, flags=D.DROP)
        yield name, _submit(dec, data, early), exp.columns
        dec.close()


def run_permissive(pos):
    def run(native, oracle, early):
        for name in ("cfg2", "sequence_example"):
            sch, rt, rows, frames, data = D.bad_block(name, 1500, 10, 9)
            full, cf = PM.with_corrupt(sch, pos)
            exp = PM.expected(oracle, data, full, rt, PM.PERM, cf)
            assert len(exp.dropped) >= 5
            dec = native.Decoder(full, rt, flags=PM.PERM, corrupt_field=cf)
            yield name, _submit(dec, data, early), exp.columns
            dec.close()
    return run


def run_permissive_all_bad(native, oracle, early):
    sch, rt, rows, frames = CORPORA["cfg2"](200, 11)
    data = b"".join(bytes(f[:-1]) + bytes([f[-1] ^ 0x10]) for f in frames)   # every payload CRC wrong
    for pos in ("middle", None):
        full, cf = PM.with_corrupt(sch, pos)
        exp = PM.expected(oracle, data, full, rt, PM.PERM, cf)
        assert len(exp.dropped) == 200
        dec = native.Decoder(full, rt, flags=PM.PERM, corrupt_field=cf)
        yield f"corrupt column {pos}", _submit(dec, data, early), exp.columns
        dec.close()


def run_resync(native, oracle, early):
    sch, rt, rows, frames = CORPORA["cfg2"](300, 12)
    for kind in ("lencrc", "garbage_random"):
        data = RS.damage(kind, frames, 13)
        for mode, flags, pos in RS.MODES:
            full, cf, dec = RS.decoder(native, sch, rt, flags, pos)
            exp = RS.expected(oracle, data, full, rt, flags, True, cf)
            assert RS.regions_of(exp), (kind, exp.spans[:4])
            yield f"{kind} {mode}", _submit(dec, data, early), exp.columns
            dec.close()


RUNS = {
    "sync_general": run_fresh("w130_general", 600, "general_path_batches"),
    "sync_tile_count": run_fresh("cfg2", 1500, "count_mode_batches"),
    "sync_tile_count_ragged": run_fresh("ragged_strings", 1500, "count_mode_batches"),
    "sync_tile_uniform": run_tile_uniform,
    "pipelined_uniform": run_pipelined("uniform", 1500),
    "pipelined_ragged": run_pipelined("ragged_strings", 1500),
    "pipelined_redone": run_redone,
    "byte_array": run_bytes,
    "no_rows": run_empty,
    "drop_malformed": run_drop,
    "permissive_column": run_permissive("middle"),
    "permissive_no_column": run_permissive(None),
    "permissive_all_bad": run_permissive_all_bad,
    "resync_lost_region": run_resync,
}


@pytest.mark.parametrize("early", [False, True], ids=["to_host", "to_host_async"])
@pytest.mark.parametrize("kind", sorted(RUNS))
def test_views(native, oracle, kind, early):
    n = 0
    for tag, b, want in RUNS[kind](native, oracle, early):
        check_readers(b, want, f"{kind} {tag}")
        b.release()
        n += 1
    assert n > 0
