"""The generated fields TFR_T_ROW_INDEX and TFR_T_RECORD_OFFSET on the GPU (include/tfrgpu.h, POSITIONS; Spark's
`_metadata.row_index`).

The expectation of a block's (row index, record offset) pairs comes from the sequential restatement of the rule
(position_walk over resync_walk's walk) and the C oracle, which tells the failing records apart (test_gpu_drop_malformed.
expected over the block's frames).  Every data column of a decode with the generated fields must be bit-identical to the same
decode without them (whose columns the other suites check against the oracle), with the same batch info and dropped list.

  1. every cases.py case and golden vector, FAILFAST / DROPMALFORMED / PERMISSIVE (with and without a corrupt-record column),
     with and without TFR_F_RESYNC;
  2. seeded corpora with failing records and damaged headers, streamed through tfr_decode_submit_at + tfr_batch_extent in
     random block cuts: exact, and independent of the cuts;
  3. every redo path, seen in the counters: learning, a shape change, malformed UTF-8, more records than provisioned, a
     pipelined framing stop under resync; a pipelined submit stays one, with no more redos than without the fields;
  4. every view: device columns, host copy, Arrow host and device export, UnsafeRows (sync, async, with partition values);
  5. placement, each kind alone, Example / SequenceExample / ByteArray, a record feature named like the field;
  6. PERMISSIVE's corrupt rows against tfr_batch_dropped plus the base; one decoder over several files;
  7. io.readFile of a multi-block file, and the C emulator of the block loop (tests/emulator/position_emulator.c)."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import partition_rows as P
import position_walk as PW
import test_gpu_batch_outputs as BO
import test_gpu_decode_rows_pipelined as RP
import test_gpu_drop_malformed as D
import test_gpu_permissive as PM
import test_gpu_resync as RS
from oracle import corpus, pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200._cabi import HostColumn
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_decode_rows import _schema_of_case
from util import assert_columns_equal

pytestmark = pytest.mark.gpu

FF = A.TFR_F_DEFAULT
DROP = A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED
PERM = A.TFR_F_DEFAULT | A.TFR_F_PERMISSIVE
RESYNC = A.TFR_F_RESYNC
RI, RO = "_tmp_metadata_row_index", "_tmp_metadata_record_offset"
KINDS = {"ri": (RI, RowIndexType), "ro": (RO, RecordOffsetType)}
INFO = ("n_rows", "n_records", "consumed_bytes", "error_code", "error_row", "error_field")
MODES = [("failfast", FF, None), ("drop", DROP, None), ("perm", PERM, "middle"), ("perm_nocol", PERM, None)]


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


# ---------------------------------------------------------------------------------------------
# schemas, the expectation, the checks
# ---------------------------------------------------------------------------------------------
def add_generated(sch, rt, where="last", kinds=("ri", "ro")):
    """-> (decoder schema, {kind: its output column}, the data fields' output columns).  ByteArray: byteArray, then the
    generated fields."""
    gens = [StructField(KINDS[k][0], KINDS[k][1](), False) for k in kinds]
    fields = list(sch.fields)
    at = len(fields) if rt == TFR_RT_BYTE_ARRAY else {"first": 0, "middle": len(fields) // 2, "last": len(fields)}[where]
    gi = {k: (1 if rt == TFR_RT_BYTE_ARRAY else at) + i for i, k in enumerate(kinds)}
    n_out = (1 if rt == TFR_RT_BYTE_ARRAY else len(fields)) + len(kinds)
    return StructType(fields[:at] + gens + fields[at:]), gi, [i for i in range(n_out) if i not in gi.values()]


def mode_of(flags):
    return PW.PERMISSIVE if flags & A.TFR_F_PERMISSIVE else PW.DROPMALFORMED if flags & A.TFR_F_DROP_MALFORMED else PW.FAILFAST


def expect(oracle, data, dsch, rt, flags, is_final=True, base=(0, 0)):
    """[(row index, record offset)] of the rows of `data` decoded at `base` with `flags`; dsch: the data fields only"""
    data = bytes(data)
    ents, _ = PW.entries(data, is_final, bool(flags & RESYNC))
    mode = mode_of(flags)
    if mode == PW.FAILFAST:
        n = oracle.decode(data, dsch, rt, flags=flags, is_final=is_final).info["n_rows"]
        return PW.positions(ents, range(n), *base)
    bad = {k for k, e in enumerate(ents) if e[0] == "region"}
    frame_at = [k for k, e in enumerate(ents) if e[0] == "frame"]
    if frame_at:
        kept = b"".join(data[e[1]:e[2]] for e in ents if e[0] == "frame")
        e = D.expected(oracle, kept, dsch, rt, (flags & A.TFR_F_VERIFY_CRC) | A.TFR_F_DROP_MALFORMED, True)
        bad |= {frame_at[i] for i, *_ in e.dropped}
    return PW.positions(ents, PW.rows(ents, bad, mode), *base)


def check_positions(cols, gi, want, what):
    n = len(want)
    for k, i in gi.items():
        c = cols[i]
        assert (c.elem_type, c.depth, c.n_rows, c.null_count) == (TFR_T_INT64, 0, n, 0), (what, k, c.elem_type, c.n_rows, c.null_count)
        assert np.unpackbits(c.validity, bitorder="little")[:n].all(), (what, k, "validity")
        got, exp = c.values[:n].tolist(), [w[0 if k == "ri" else 1] for w in want]
        if got != exp:
            r = next(r for r in range(n) if got[r] != exp[r])
            raise AssertionError(f"{what} {k}: row {r} of {n}: {got[r]} != {exp[r]}")


def positions_of(cols, gi, n):
    return list(zip(cols[gi["ri"]].values[:n].tolist(), cols[gi["ro"]].values[:n].tolist()))


def check_same_data(bg, bp, didx, what):
    """a decode with the generated fields is the decode without them, plus those columns"""
    assert {k: bg.info[k] for k in INFO} == {k: bp.info[k] for k in INFO}, what
    assert bg.dropped_spans() == bp.dropped_spans(), what
    got = bg.to_host()
    assert_columns_equal([got[i] for i in didx], bp.to_host(), None, what)
    return got


def extent_want(b, flags, data, is_final):
    """tfr_batch_extent: the walk's consumed bytes and entries; a FAILFAST error ends them in front of its record"""
    if b.info["error_code"]:
        return b.info["consumed_bytes"], b.info["error_row"]
    ents, consumed = PW.entries(bytes(data), is_final, bool(flags & RESYNC))
    return consumed, len(ents)


def pair(native, full, rt, flags, cf=None, where="last", kinds=("ri", "ro")):
    """(decoder without the generated fields, decoder with them, {kind: column}, data columns)"""
    gsch, gi, didx = add_generated(full, rt, where, kinds)
    plain = native.Decoder(full, rt, flags=flags, corrupt_field=cf)
    gen = native.Decoder(gsch, rt, flags=flags, corrupt_field=None if cf is None else didx[cf])
    return plain, gen, gi, didx


# ---------------------------------------------------------------------------------------------
# 1. every case and golden vector, every mode
# ---------------------------------------------------------------------------------------------
def _inputs():
    import cases as CS
    import test_golden as G
    for c in CS.all_cases():
        yield c.name, c.data(), _schema_of_case(c), c.record_type, getattr(c, "flags", FF), getattr(c, "is_final", True)
    for e in G.INDEX:
        sch = byte_array_schema() if e["record_type"] == 2 else G.schema_of(e)
        yield e["name"], open(os.path.join(G.HERE, e["file"]), "rb").read(), sch, e["record_type"], e["flags"], e["is_final"]


# TFR_F_RESYNC needs DROPMALFORMED or PERMISSIVE
MODES_RESYNC = [m + (r,) for r in (False, True) for m in MODES if not (r and m[0] == "failfast")]
MODE_IDS = [m[0] + ("/resync" if m[3] else "") for m in MODES_RESYNC]


@pytest.mark.parametrize("mode, mflags, pos, resync", MODES_RESYNC, ids=MODE_IDS)
def test_every_case_and_golden_vector(native, oracle, mode, mflags, pos, resync):
    base = (7, 3 << 32)
    n = n_bad = 0
    for name, data, dsch, rt, cflags, is_final in _inputs():
        flags = cflags | mflags | (RESYNC if resync else 0)
        if (resync and not flags & A.TFR_F_VERIFY_CRC) or (flags & A.TFR_F_PERMISSIVE and rt == TFR_RT_BYTE_ARRAY):
            continue
        full, cf = PM.with_corrupt(dsch, pos) if flags & A.TFR_F_PERMISSIVE else (dsch, None)
        plain, gen, gi, didx = pair(native, full, rt, flags, cf)
        what = f"{name}/{mode}{'/resync' if resync else ''}"
        try:
            bp, _ = plain.decode(data, is_final=is_final)
            bg, used = gen.decode(data, is_final=is_final, first_entry=base[0], first_offset=base[1])
            got = check_same_data(bg, bp, didx, what)
            check_positions(got, gi, expect(oracle, data, dsch, rt, flags, is_final, base), what)
            assert bg.extent() == extent_want(bg, flags, data, is_final), what
            n += 1
            n_bad += len(bg.dropped())
            bg.release(); bp.release()
        finally:
            plain.close(); gen.close()
    assert n > 50 and (mode == "failfast" or n_bad > 10), (n, n_bad)


# ---------------------------------------------------------------------------------------------
# 2. seeded corpora, streamed in random block cuts
# ---------------------------------------------------------------------------------------------
def damaged(frames, seed, n_bad, n_hdr):
    """the frames with a payload bit flipped in n_bad of them (a data CRC error) and a length-CRC bit in n_hdr others"""
    R_ = random.Random(seed)
    fr = list(frames)
    at = R_.sample(range(1, len(fr) - 1), n_bad + n_hdr)
    for i in at[:n_bad]:
        f = bytearray(fr[i])
        if len(f) > 16:
            f[12 + R_.randrange(len(f) - 16)] ^= 1 << R_.randrange(8)
        fr[i] = bytes(f)
    for i in at[n_bad:]:
        fr[i] = RS.flip_lencrc(fr[i], R_)
    return b"".join(fr)


def stream(dec, data, cuts, gi):
    """the block loop of a streaming reader: each block submitted at the extents of the ones before it -> every row's positions"""
    data = bytes(data)
    out, pos, ent, i = [], 0, 0, 0
    cuts = sorted(set(c for c in cuts if 0 < c < len(data))) + [len(data)]
    while True:
        while cuts[i] <= pos:
            i += 1
        stop = cuts[i]
        final = stop == len(data)
        b = dec.submit(data[pos:stop], is_final=final, first_entry=ent, first_offset=pos)
        used, n = b.extent()
        out += positions_of(b.to_host(), gi, b.n_rows)
        err = b.info["error_code"]
        b.release()
        if err or final:
            return out
        if used == 0:
            i += 1
            continue
        pos += used
        ent += n


STREAMED = [(name,) + m for name in ("cfg2", "sequence_example", "byte_array") for m in MODES_RESYNC
            if not (name == "byte_array" and m[0].startswith("perm"))]          # PERMISSIVE takes no ByteArray records


@pytest.mark.parametrize("name, mode, mflags, pos, resync", STREAMED,
                         ids=[f"{s[0]}/{s[1]}" + ("/resync" if s[4] else "") for s in STREAMED])
def test_streamed_in_random_cuts(native, oracle, name, mode, mflags, pos, resync):
    flags = mflags | (RESYNC if resync else 0)
    seed = 31 + len(name) + len(mode) + resync
    sch, rt, _, frames = D.CORPORA[name](1200, seed)
    data = damaged(frames, seed, 0 if mode == "failfast" else 8, 3 if resync else 0)
    full, cf = PM.with_corrupt(sch, pos) if flags & A.TFR_F_PERMISSIVE else (sch, None)
    gsch, gi, didx = add_generated(full, rt, "middle")
    want = expect(oracle, data, sch, rt, flags)
    assert len(want) > 1000
    if mode == "failfast":
        assert [w[0] for w in want] == list(range(1200))
    dec = native.Decoder(gsch, rt, flags=flags, corrupt_field=None if cf is None else didx[cf])
    try:
        R_ = random.Random(seed)
        for rnd in range(4):
            k = R_.randrange(2, 12)
            cuts = sorted(R_.sample(range(1, len(data)), k))
            assert stream(dec, data, cuts, gi) == want, (name, mode, rnd, cuts)
        if name == "cfg2":
            assert dec.stats()["speculative_submits"] > 0, dec.stats()
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# 3. every redo path: the batch keeps its base, and the pipeline is the one without the fields
# ---------------------------------------------------------------------------------------------
def _encode_rows(sch, rows):
    import wire_rewrite as W
    return b"".join(pyref.frame_fast(W.canonical(sch, row)) for row in rows)


def _uniform(n, seed, float_len):
    sch, cols = corpus.cfg2_columns(n, seed=seed, n_bytes=0, float_len=float_len)
    return sch, _encode_rows(sch, [tuple(c.get(r) for c in cols) for r in range(n)])


def _redo_path(oracle, path):
    """-> (schema, flags, learning blocks, the block that takes the redo path, the counter that shows it)"""
    if path == "learning":
        sch, data = _uniform(800, 1, 8)
        return sch, FF, [], data, "count_mode_batches"
    if path == "shape_change":
        sch, learn = _uniform(800, 2, 8)
        return sch, FF, [learn] * 3, _uniform(800, 3, 5)[1], "speculative_redone"
    rng = np.random.default_rng(4)
    if path == "malformed_utf8":
        lens = rng.integers(5, 40, 3000)
        return RP.STR_SCH, FF, [RP._strings(oracle, lens, 11)] * 3, RP._strings(oracle, lens, 11, bad={17, 1500}), "transcode_reruns"
    if path == "more_records":
        return (RP.STR_SCH, FF, [RP._strings(oracle, rng.integers(190, 211, 2000), 7)] * 3,
                RP._strings(oracle, rng.integers(10, 30, 6000), 8), "speculative_redone")
    assert path == "framing_stop"
    sch, rt, _, frames = D.CORPORA["cfg2"](1500, 5)
    return sch, DROP | RESYNC, [b"".join(frames)] * 3, damaged(frames, 5, 4, 2), "lost_regions"


@pytest.mark.parametrize("path", ["learning", "shape_change", "malformed_utf8", "more_records", "framing_stop"])
def test_redo_paths_keep_the_base(native, oracle, path):
    sch, flags, learn, block, counter = _redo_path(oracle, path)
    plain, gen, gi, didx = pair(native, sch, TFR_RT_EXAMPLE, flags, where="first")
    base = (1 << 20, (1 << 40) + 3)
    try:
        for blk in learn:
            for d in (plain, gen):
                d.submit(blk).release()
        s0 = gen.stats()
        bp = plain.submit(block)
        bp.unsafe_rows_async(True)
        bg = gen.submit(block, first_entry=base[0], first_offset=base[1])
        bg.unsafe_rows_async(True)
        got = check_same_data(bg, bp, didx, path)
        want = expect(oracle, block, sch, TFR_RT_EXAMPLE, flags, True, base)
        check_positions(got, gi, want, path)
        exp = D.Expect(expected_columns(bp.to_host(), gi, didx, want), {"n_rows": len(want)}, [])
        D.check_rows(bg, long_schema(add_generated(sch, TFR_RT_EXAMPLE, "first")[0]), exp, None, f"{path} rows (async)")
        bp.release(); bg.release()
        sp, sg = plain.stats(), gen.stats()
        assert sp == sg, (path, sp, sg)          # the same batches took the same paths, redos included
        assert D.delta(s0, sg)[counter] > 0, (path, s0, sg)
        if path != "learning":
            assert sg["speculative_submits"] > 0, sg
        # after the redo the next block is submitted without a host synchronisation again, and keeps its base
        for d in (plain, gen):
            s0 = d.stats()
            kw = {"first_entry": base[0], "first_offset": base[1]} if d is gen else {}
            b = d.submit(block, **kw)
            b.wait()
            if d is gen:
                check_positions(b.to_host(), gi, expect(oracle, block, sch, TFR_RT_EXAMPLE, flags, True, base), f"{path} after")
            b.release()
            delta = D.delta(s0, d.stats())
            if path not in ("learning", "framing_stop"):
                assert delta["speculative_submits"] == 1, (path, delta)
        assert plain.stats() == gen.stats(), path
    finally:
        plain.close(); gen.close()


# ---------------------------------------------------------------------------------------------
# 4. every view of the generated columns
# ---------------------------------------------------------------------------------------------
class ArrowSchema(C.Structure):
    _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64), ("n_children", C.c_int64),
                ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowArray(C.Structure):
    _fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64), ("n_children", C.c_int64),
                ("buffers", C.POINTER(C.c_void_p)), ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p),
                ("private_data", C.c_void_p)]


class ArrowDeviceArray(C.Structure):
    _fields_ = [("array", ArrowArray), ("device_id", C.c_int64), ("device_type", C.c_int32), ("sync_event", C.c_void_p),
                ("reserved", C.c_int64 * 3)]


_RELEASE = C.CFUNCTYPE(None, C.c_void_p)


def arrow_device_column(native, b, col):
    """tfr_batch_export_arrow_device of one int64 column -> (format, null count, values copied from the device)"""
    da, sc = ArrowDeviceArray(), ArrowSchema()
    native._check(native.lib().tfr_batch_export_arrow_device(b.h, col, C.addressof(da), C.addressof(sc)))
    try:
        assert da.device_type == 2 and da.array.n_buffers == 2
        vals = BO._dev_array(da.array.buffers[1], da.array.length, np.int64)
        return sc.format.decode(), da.array.null_count, vals
    finally:
        _RELEASE(da.array.release)(C.addressof(da.array))
        _RELEASE(sc.release)(C.addressof(sc))


def long_schema(gsch):
    """the decoder schema as Spark sees it: a generated field is a non-nullable LongType"""
    return StructType([StructField(f.name, LongType(), False) if isinstance(f.dataType, (RowIndexType, RecordOffsetType)) else f
                       for f in gsch])


def expected_columns(data_cols, gi, didx, want):
    n = len(want)
    cols = [None] * (len(didx) + len(gi))
    for j, i in enumerate(didx):
        cols[i] = data_cols[j]
    for k, i in gi.items():
        cols[i] = HostColumn(TFR_T_INT64, 0, n, np.packbits(np.ones(n, np.uint8), bitorder="little"), [],
                             np.array([w[0 if k == "ri" else 1] for w in want], np.int64))
    return cols


def check_views(native, b, gsch, want_cols, gi, what, async_rows):
    assert_columns_equal(BO.device_columns(b), want_cols, None, f"{what} device columns")
    assert_columns_equal(b.to_host(), want_cols, None, f"{what} host copy")
    BO.check_arrow(b.to_arrow(), want_cols, f"{what} arrow host")
    for i in gi.values():
        fmt, nulls, vals = arrow_device_column(native, b, i)
        assert fmt == "l" and nulls == 0 and np.array_equal(vals, want_cols[i].values), f"{what} arrow device col {i}"
    exp = D.Expect(want_cols, {"n_rows": want_cols[0].n_rows}, [])
    D.check_rows(b, long_schema(gsch), exp, None, f"{what} rows{' (async)' if async_rows else ''}")


@pytest.mark.parametrize("name, flags", [("cfg2", FF), ("byte_array", FF), ("cfg2_perm", PERM | RESYNC)])
def test_every_view(native, oracle, name, flags):
    sch, rt, _, frames = D.CORPORA[name.split("_perm")[0]](1500, 9)
    data = b"".join(frames) if flags == FF else damaged(frames, 9, 5, 2)
    full, cf = PM.with_corrupt(sch, "last") if flags & A.TFR_F_PERMISSIVE else (sch, None)
    plain, gen, gi, didx = pair(native, full, rt, flags, cf, where="middle")
    gsch = add_generated(full, rt, "middle")[0]
    base = (11, 1 << 33)
    want = expect(oracle, data, sch, rt, flags, True, base)
    try:
        for it in range(4):                        # the synchronous first batches, then pipelined ones
            async_rows = it % 2 == 1
            bp, _ = plain.decode(data)
            b = gen.submit(data, first_entry=base[0], first_offset=base[1])
            if async_rows:
                b.unsafe_rows_async(True)
            if flags == FF and it == 0:
                assert_columns_equal(bp.to_host(), oracle.decode(data, sch, rt).columns, None, "plain vs oracle")
            cols = expected_columns(bp.to_host(), gi, didx, want)
            check_views(native, b, gsch, cols, gi, f"{name} #{it}", async_rows)
            if it == 3:                             # partition values appended
                pr = (P.partition_row(*D.PART), P.var_flags(D.PART[0]))
                b2 = gen.submit(data, first_entry=base[0], first_offset=base[1])
                b2.unsafe_rows_async(True, pr)
                D.check_rows(b2, long_schema(gsch), D.Expect(cols, {"n_rows": len(want)}, []), D.PART, f"{name} partitioned rows")
                b2.release()
            b.release(); bp.release()
        if flags == FF and name == "cfg2":
            assert gen.stats()["speculative_submits"] >= 2 and gen.stats()["rows_async"] >= 1, gen.stats()
    finally:
        plain.close(); gen.close()


# ---------------------------------------------------------------------------------------------
# 5. placement, each kind alone, the record types, a feature named like the field
# ---------------------------------------------------------------------------------------------
# ByteArray puts the generated fields behind byteArray
PLACED = [(name, where) for name in ("cfg2", "sequence_example", "byte_array") for where in ("first", "middle", "last")
          if name != "byte_array" or where == "last"]


@pytest.mark.parametrize("kinds", [("ri", "ro"), ("ri",), ("ro",), ("ro", "ri")], ids=["both", "row_index", "record_offset", "reversed"])
@pytest.mark.parametrize("name, where", PLACED, ids=[f"{n}/{w}" for n, w in PLACED])
def test_placement_kinds_and_record_types(native, oracle, name, where, kinds):
    sch, rt, _, frames = D.CORPORA[name](900, 13)
    data = b"".join(frames)
    plain, gen, gi, didx = pair(native, sch, rt, FF, None, where, kinds)
    want = expect(oracle, data, sch, rt, FF, True, (3, 5))
    try:
        for it in range(3):
            bp, _ = plain.decode(data)
            bg = gen.submit(data, first_entry=3, first_offset=5)
            check_positions(check_same_data(bg, bp, didx, f"{name}/{where}/{kinds} #{it}"), gi, want, f"{name}/{where}/{kinds}")
            bg.release(); bp.release()
    finally:
        plain.close(); gen.close()


def _entry(key, feature_bytes):
    k = key.encode()
    body = b"\x0a" + bytes([len(k)]) + k + b"\x12" + bytes([len(feature_bytes)]) + feature_bytes
    return b"\x0a" + bytes([len(body) + 2]) + b"\x0a" + bytes([len(body)]) + body       # one more Features occurrence (merges)


@pytest.mark.parametrize("flags", [FF, DROP], ids=["failfast", "drop"])
def test_a_record_feature_named_like_the_field_is_ignored(native, oracle, flags):
    """never looked up: a long, a bytes list of the wrong kind under the name; still validated: a malformed one fails the
    record exactly as it does for a decoder without the field in its schema"""
    sch = StructType([StructField("a", LongType()), StructField("s", StringType())])
    payloads = []
    for i in range(300):
        feats = {"a": pyref.int64_feature(i), "s": pyref.bytes_feature(f"v{i}")}
        if i % 3 == 0:
            feats[RI] = pyref.int64_feature(-5)
        if i % 3 == 1:
            feats[RO] = pyref.bytes_feature("not a long")
        p = pyref.example(feats).SerializeToString()
        if i == 250:
            p += _entry(RI, b"\x1a\x05\x0a\x09")             # an Int64List whose packed values run past the message
        payloads.append(p)
    data = b"".join(pyref.frame(p) for p in payloads)
    assert oracle.decode(data, StructType([StructField(RO, LongType())] + list(sch)), 0).info["error_code"] == A.TFR_E_KIND_MISMATCH   # they are there
    plain, gen, gi, didx = pair(native, sch, TFR_RT_EXAMPLE, flags, None, "middle")
    try:
        bp, _ = plain.decode(data)
        bg, _ = gen.decode(data, first_entry=2, first_offset=9)
        got = check_same_data(bg, bp, didx, "named like the field")
        want = expect(oracle, data, sch, 0, flags, True, (2, 9))
        check_positions(got, gi, want, "named like the field")
        assert len(want) == (250 if flags == FF else 299)
    finally:
        plain.close(); gen.close()


# ---------------------------------------------------------------------------------------------
# 6. PERMISSIVE's corrupt rows; one decoder over several files
# ---------------------------------------------------------------------------------------------
def test_permissive_corrupt_rows_are_the_dropped_list_plus_the_base(native, oracle):
    sch, rt, _, frames = D.CORPORA["cfg2"](1000, 21)
    data = damaged(frames, 21, 9, 3)
    full, cf = PM.with_corrupt(sch, "first")
    gsch, gi, didx = add_generated(full, rt, "last")
    dec = native.Decoder(gsch, rt, flags=PERM | RESYNC, corrupt_field=didx[cf])
    try:
        base = (1000, 123456789)
        b, _ = dec.decode(data, first_entry=base[0], first_offset=base[1])
        cols = b.to_host()
        pos = positions_of(cols, gi, b.n_rows)
        dropped = b.dropped()
        assert len(dropped) >= 9 and any(code in A.FRAMING_ERRORS for _, _, code, _ in dropped)
        corrupt = cols[didx[cf]]
        for rec, off, _, _ in dropped:
            assert pos[rec] == (base[0] + rec, base[1] + off) and corrupt.valid(rec)
        assert [p[0] for p in pos] == list(range(base[0], base[0] + b.n_rows))
        check_positions(cols, gi, expect(oracle, data, sch, rt, PERM | RESYNC, True, base), "permissive")
        b.release()
    finally:
        dec.close()


def test_one_decoder_over_several_files(native, oracle):
    """each file starts at (0, 0); a pipelined decoder carries nothing from one file into the next"""
    dec = None
    try:
        for k, (name, n) in enumerate([("cfg2", 700), ("cfg2", 1300), ("cfg2", 900)]):
            sch, rt, _, frames = D.CORPORA[name](n, 40 + k)
            data = damaged(frames, 40 + k, 4, 0)
            gsch, gi, _ = add_generated(sch, rt, "first")
            dec = dec or native.Decoder(gsch, rt, flags=DROP)
            for rep in range(2):
                b = dec.submit(data)
                check_positions(b.to_host(), gi, expect(oracle, data, sch, rt, DROP), f"file {k} #{rep}")
                b.release()
    finally:
        if dec:
            dec.close()


def test_negative_base_is_refused(native):
    sch, rt, _, frames = D.CORPORA["cfg2"](50, 1)
    gsch, _, _ = add_generated(sch, rt)
    dec = native.Decoder(gsch, rt)
    try:
        for fe, fo in [(-1, 0), (0, -1)]:
            with pytest.raises(native.TfrError) as e:
                dec.submit(b"".join(frames), first_entry=fe, first_offset=fo)
            assert e.value.code == A.TFR_E_INVALID_ARG
        assert dec.stats()["batches"] == 0
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# 7. io.readFile of a multi-block file
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["FAILFAST", "DROPMALFORMED"])
def test_read_file_row_index(native, oracle, tmp_path, mode):
    from spark_tfrecord_b200 import io as tio
    sch, rt, _, frames = D.CORPORA["cfg2"](3000, 17)
    data = b"".join(frames) if mode == "FAILFAST" else damaged(frames, 17, 12, 0)
    path = tmp_path / "part-00000.tfrecord"
    path.write_bytes(data)
    req = StructType([StructField(RI, LongType(), False), sch.fields[0], StructField(RO, LongType(), False)])
    rows = list(tio.TFRecordFileReader.readFile(None, {"mode": mode}, tio.PartitionedFile(str(path)), req, block_bytes=256 << 10))
    want = expect(oracle, data, sch, rt, FF if mode == "FAILFAST" else DROP)
    assert [(r[0], r[2]) for r in rows] == want
    if mode == "FAILFAST":
        assert [r[0] for r in rows] == list(range(3000))
    else:
        assert len(rows) == 3000 - 12
    assert len(data) > 4 * (256 << 10)


@pytest.mark.parametrize("mode", [0, 1], ids=["failfast", "drop"])
def test_emulated_block_loop_with_positions(native, oracle, tmp_path, mode):
    """the plain-C BlockIterator (tfr_decode_submit_at, tfr_batch_extent, UnsafeRows) over a file the C writer wrote, with
    failing records in DROPMALFORMED; every block size gives the whole file's positions"""
    import subprocess
    from test_encode_pipeline_host import build_emulator, emulator_schema
    from test_row_index_host import build_position_emulator
    writer = build_emulator(str(tmp_path / "rowwrite"))
    reader = build_position_emulator(str(tmp_path / "positions"))
    p = subprocess.run([writer, "rowwrite", str(tmp_path), "20000", "4000"], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    path = os.path.join(str(tmp_path), "part-00000.tfrecord")
    data = open(path, "rb").read()
    if mode:
        frames, o = [], 0
        while o < len(data):
            L = int.from_bytes(data[o:o + 8], "little")
            frames.append(data[o:o + 16 + L])
            o += 16 + L
        data = damaged(frames, 3, 10, 0)
        path = str(tmp_path / "bad.tfrecord")
        open(path, "wb").write(data)
    want = expect(oracle, data, emulator_schema(), 0, DROP if mode else FF)
    assert len(want) == 20000 - 10 * mode
    for block in (4096, 1 << 20, 64 << 20):
        p = subprocess.run([reader, "positions", path, str(block), str(mode)], capture_output=True, text=True, timeout=900)
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr
        lines = p.stdout.splitlines()
        assert lines[-1] == f"status 0 row -1 rows {len(want)}", (block, lines[-1])
        assert [tuple(map(int, l.split())) for l in lines[:-1]] == want, block
