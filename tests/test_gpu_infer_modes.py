"""Schema inference in DROPMALFORMED and PERMISSIVE on the GPU (tfr_infer_create_mode, infer_kernel<true>) against
`infer_modes_oracle.infer_mode`, whose tolerant inference tests/test_infer_modes_host.py pins on the CPU.

Every case is inferred three ways -- the bytes in host memory, a device tensor at an odd address, and `update_block`
over random splits -- and each must give the oracle's status, its {name: code} map and its skipped list
(frame index, frame offset, code), the split's lists put back into whole-buffer numbering.  After a framing error the
map is the one the records before the stop merged.  Cases: the seeded corpora with the corrupt-record column's name
planted; record atomicity, with maps of fewer and of more than 32 entries (a record over several flushes of the warp);
all-bad blocks and framing errors after skipped records; the device-table limits; FAILFAST through the new entry point
against tfr_infer_create; PERMISSIVE's name in every place and kind; and io.DefaultSource.inferSchema end to end."""
import logging
import os
import random

import numpy as np
import pytest

import infer_corpus as C
import infer_modes_oracle as M
import test_gpu_permissive as P
from oracle import pyref
from oracle.pyref import ld, map_entry
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import BinaryType, FloatType, LongType, StringType, StructField, StructType
from test_gpu_infer_fuzz import _blocks, _on_device_odd, native  # noqa: F401  (native: the fixture)
from test_infer_modes_host import CORRUPT, DROP, PERM, framed, plant, planted_value

pytestmark = pytest.mark.gpu
FRAMING = (A.TFR_E_CRC_LENGTH, A.TFR_E_TRUNCATED, A.TFR_E_RECORD_TOO_LARGE)
MODES = [(DROP, None), (PERM, CORRUPT)]


def _frame_starts(data: bytes):
    """byte offsets of the frames whose headers can be read (length CRC not checked): where a block split may count them"""
    starts, pos = [], 0
    while len(data) - pos >= 12:
        starts.append(pos)
        pos += 16 + int.from_bytes(data[pos:pos + 8], "little")
    return starts


def _framing_stop(data: bytes) -> int:
    """the offset at which the frame chain stops (a bad length CRC, a length over 2 GiB, a truncated frame)"""
    pos = 0
    while len(data) - pos >= 12:
        n = int.from_bytes(data[pos:pos + 8], "little")
        if pyref.masked_crc32c(data[pos:pos + 8]) != int.from_bytes(data[pos + 8:pos + 12], "little") or n > 0x7FFFFFFF \
                or len(data) - pos < 16 + n:
            break
        pos += 16 + n
    return pos


def _result(native, inf):
    try:
        return inf.result()
    except native.TfrError as e:
        return e.code                                               # the ArrayType(ArrayType(null)) conflict


def _run(native, rt, flags, name, feed):
    """-> (status, names -> codes or None, skipped [(frame index, offset, code)]); `feed(inf, skipped)` makes the calls.
    After a framing error the map is what the records before the stop merged (or the status of its merge conflict)."""
    inf = native.Infer(rt, 0, flags, name)
    skipped = []
    try:
        try:
            feed(inf, skipped)
        except native.TfrError as e:
            return e.code, (_result(native, inf) if e.code in FRAMING else None), skipped
        r = _result(native, inf)
        return (r, None, skipped) if isinstance(r, int) else (0, r, skipped)
    finally:
        inf.close()


def _whole(inf, data, skipped):
    try:
        inf.update(data)
    finally:
        skipped += [(r, o, c) for r, o, c, _ in inf.skipped()]


def _split(data: bytes, R: random.Random):
    """update_block over random blocks: tiny ones, ends inside a header and inside a payload"""
    starts = _frame_starts(data)

    def feed(inf, skipped):
        pos = 0
        while True:
            cut = R.choice(["tiny", "header", "payload", "big"])
            nxt = [s for s in starts if s > pos]
            if cut == "tiny":
                end = pos + R.randrange(1, 40)
            elif cut == "header" and nxt:
                end = nxt[0] + R.randrange(1, 12)
            elif cut == "payload" and len(nxt) > 1:
                end = nxt[1] - R.randrange(1, 5)
            else:
                end = pos + R.randrange(1, 1 << 16)
            end = max(pos + 1, min(end, len(data)))
            final = end == len(data)
            base = sum(1 for s in starts if s < pos)
            try:
                used = inf.update_block(data[pos:end], final)
            finally:
                skipped += [(base + r, pos + o, c) for r, o, c, _ in inf.skipped()]
            pos += used
            if final:
                return
    return feed


def check(native, oracle, data: bytes, rt: int, flags: int, name, R: random.Random, what: str):
    """the three ways against the oracle; -> the oracle's (status, map, skipped)"""
    rc, codes, skipped = M.infer_mode(data, rt, flags, name)
    if rc in FRAMING:                                               # the records before the stop, merged
        prc, pcodes, _ = M.infer_mode(data[:_framing_stop(data)], rt, flags, name)
        codes = pcodes if prc == 0 else prc
    want = (rc, codes if rc == 0 or rc in FRAMING else None, skipped)
    msg = f"{what} ({'PERMISSIVE' if name else 'DROPMALFORMED'})"
    got = _run(native, rt, flags, name, lambda inf, s: _whole(inf, np.frombuffer(data, np.uint8), s))
    assert got == want, f"update (host): {got} != {want}; {msg}"
    got = _run(native, rt, flags, name, lambda inf, s: _whole(inf, _on_device_odd(data), s))
    assert got == want, f"update (device, odd address): {got} != {want}; {msg}"
    if data:
        got = _run(native, rt, flags, name, _split(data, R))
        assert got == want, f"update_block: {got} != {want}; {msg}"
    return want


# --------------------------------------------------------------------------------------------
# 3. the seeded corpora
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rt", [0, 1])
def test_seeded_corpora_match_the_oracle(native, oracle, rt):
    R = random.Random(10 + rt)
    seen, n_skipped = set(), 0
    for seed in range(48):
        b = C.batch(seed, rt, R.choice([1, 2, 33, 64, 200]))
        payloads = [plant(R, rt, p) if R.random() < 0.2 else p for p in b.payloads]
        crc = [b.crc_row] if b.crc_row is not None else []
        data = framed(payloads, crc, truncated=b.truncated)
        for flags, name in MODES:
            rc, _, skipped = check(native, oracle, data, rt, flags, name, R, f"seed {seed}: {b.describe()}")
            seen.add(rc)
            n_skipped += len(skipped)
    assert {0, A.TFR_E_TRUNCATED} <= seen and n_skipped > 20, (seen, n_skipped)


# --------------------------------------------------------------------------------------------
# 4. record atomicity
# --------------------------------------------------------------------------------------------
def _fill(k: int, tag: bytes = b"f", m: int = 0):
    """k clean entries of map m (0: features / context, 1: feature_lists)"""
    return b"".join(map_entry(tag + b"%03d" % i, C.fl(C.i64(i)) if m else C.i64(i)) for i in range(k))


def _flfill(k: int):
    return b"".join(map_entry(b"l%03d" % i, C.fl(C.i64(i))) for i in range(k))


@pytest.mark.parametrize("pad", [3, 45])
def test_a_failing_record_contributes_nothing(native, oracle, pad):
    R = random.Random(pad)
    clean = ld(1, _fill(pad) + map_entry(b"k", C.i64(1)))
    cases = {
        # a name that only a failing record carries is absent; the failing record's value error sits after it
        "name_only_in_a_failing_record": (0, [clean, ld(1, map_entry(b"only_bad", C.i64(1)) + _fill(pad) + map_entry(b"x", C.UNSET))]),
        # a failing record does not raise a name's code (k: Long here, array of Long in the failing one)
        "no_raised_code": (0, [clean, ld(1, map_entry(b"k", C.i64(1, 2)) + _fill(pad, b"g") + map_entry(b"y", C.UNSET))]),
        # the failing record first, then a clean one
        "failing_first": (0, [ld(1, _fill(pad, b"h") + map_entry(b"k", C.f32(1.0, 2.0))) + b"\x0a\x05\x01", clean]),
        # a value error in an entry that a later one of the same key overwrites is no failure
        "overwritten_error": (0, [ld(1, map_entry(b"a", C.UNSET) + _fill(pad) + map_entry(b"a", C.i64(1)))]),
        # SequenceExample: clean context, failing feature_lists (empty FeatureList / a step whose kind is not set / malformed)
        "seq_clean_context_empty_flist": (1, [ld(1, map_entry(b"ctx_only", C.i64(1)) + _fill(pad)) + ld(2, _flfill(pad) + map_entry(b"e", b"")),
                                              ld(1, map_entry(b"k", C.i64(1)))]),
        "seq_clean_context_unset_step": (1, [ld(1, map_entry(b"k", C.i64(1, 2)) + _fill(pad)) + ld(2, map_entry(b"s", C.fl(C.i64(1), C.UNSET)) + _flfill(pad)),
                                             ld(1, map_entry(b"k", C.i64(1)))]),
        "seq_clean_context_malformed_flist": (1, [ld(2, _flfill(pad)) + ld(1, map_entry(b"ctx_only", C.i64(1)) + _fill(pad)) + ld(2, b"\x0a\x05\x01")]),
        # ArrayType(ArrayType(null)) against another type: only a skipped record brings the conflict
        "conflict_only_from_a_skipped_record": (1, [ld(2, map_entry(C.EMPTY_STEPS[0], C.fl(C.i64(1))) + _flfill(pad)),
                                                    ld(2, map_entry(C.EMPTY_STEPS[0], C.fl(C.i64(), C.f32())) + _flfill(pad)) + ld(1, map_entry(b"z", C.UNSET))]),
        "conflict_only_from_a_crc_failure": (1, [ld(2, map_entry(C.EMPTY_STEPS[0], C.fl(C.i64(1)))),
                                                 ld(2, map_entry(C.EMPTY_STEPS[0], C.fl(C.i64()))) + ld(1, _fill(pad))]),
    }
    for what, (rt, ps) in cases.items():
        crc = [1] if what == "conflict_only_from_a_crc_failure" else []
        data = framed(ps, crc)
        for flags, name in MODES:
            rc, codes, skipped = check(native, oracle, data, rt, flags, name, R, f"{what}, pad {pad}")
            assert rc == 0, what
            if what == "name_only_in_a_failing_record":
                assert b"only_bad" not in codes and codes[b"k"] == 1 and [s[0] for s in skipped] == [1]
            elif what == "no_raised_code":
                assert codes[b"k"] == 1 and b"g000" not in codes and [s[0] for s in skipped] == [1]
            elif what == "failing_first":
                assert codes[b"k"] == 1 and b"h000" not in codes and skipped == [(0, 0, A.TFR_E_MALFORMED_PROTO)]
            elif what == "overwritten_error":
                assert codes[b"a"] == 1 and skipped == []
            elif what.startswith("seq_clean_context"):
                assert b"ctx_only" not in codes and b"f000" not in codes and b"l000" not in codes and [s[0] for s in skipped] == [0]
                if what != "seq_clean_context_malformed_flist":
                    assert codes[b"k"] == 1
            else:
                assert codes[C.EMPTY_STEPS[0]] == 7 and [s[0] for s in skipped] == [1]


# --------------------------------------------------------------------------------------------
# 5. all bad; framing errors after skipped records
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rt", [0, 1])
def test_every_record_bad(native, oracle, rt):
    R = random.Random(rt)
    bad = [ld(1, map_entry(b"k%d" % i, C.UNSET)) if i % 3 == 0 else ld(1, _fill(i % 50)) + b"\x0a\x05\x01" if i % 3 == 1
           else ld(1, map_entry(b"c%d" % i, C.i64(i))) for i in range(300)]
    data = framed(bad, [i for i in range(300) if i % 3 == 2])
    for flags, name in MODES:
        rc, codes, skipped = check(native, oracle, data, rt, flags, name, R, "every record bad")
        assert rc == 0 and codes == {} and [s[0] for s in skipped] == list(range(300))


@pytest.mark.parametrize("rt", [0, 1])
def test_framing_errors_after_skipped_records(native, oracle, rt):
    R = random.Random(20 + rt)
    ps = C.batch(3, rt, 60, mode="clean").payloads
    for r in (2, 17, 40):
        ps[r] = ld(1, map_entry(b"bad%d" % r, C.UNSET))
    for damage, data in (("truncated", framed(ps, truncated=True)), ("length CRC", framed(ps, lencrc_row=50))):
        fail_rc = _run(native, rt, 0, None, lambda inf, s: inf.update(data))[0]
        for flags, name in MODES:
            rc, _, skipped = check(native, oracle, data, rt, flags, name, R, damage)
            assert rc == (A.TFR_E_TRUNCATED if damage == "truncated" else A.TFR_E_CRC_LENGTH)
            assert [s[0] for s in skipped] == [2, 17, 40]
        # FAILFAST stops at the first failing record, before the framing error
        assert fail_rc == A.TFR_E_KIND_MISMATCH
        clean = [p for r, p in enumerate(ps) if r not in (2, 17, 40)]
        d2 = framed(clean, truncated=True) if damage == "truncated" else framed(clean, lencrc_row=47)
        assert _run(native, rt, 0, None, lambda inf, s: inf.update(d2))[0] == rc


# --------------------------------------------------------------------------------------------
# 6. limits
# --------------------------------------------------------------------------------------------
def test_limits(native, oracle):
    wide = ld(1, _fill(1025))
    clean = ld(1, map_entry(b"k", C.i64(1)))
    for flags, name in MODES:
        for rt in (0, 1):
            got = _run(native, rt, flags, name, lambda inf, s: _whole(inf, pyref.frame_fast(wide), s))
            assert got[0] == A.TFR_E_BATCH_TOO_LARGE and got[2] == []
            # a value error among the entries: the entries past the window decide, so it still fails the call
            p = ld(1, map_entry(b"f000", C.UNSET) + _fill(1025)[len(map_entry(b"f000", C.i64(0))):])
            assert _run(native, rt, flags, name, lambda inf, s: inf.update(pyref.frame_fast(p)))[0] == A.TFR_E_BATCH_TOO_LARGE
            # over the limit and malformed, or over the limit with a flipped data CRC: skipped
            for what, data in (("malformed", framed([clean, wide + b"\x0a\x05\x01", clean])), ("crc", framed([clean, wide, clean], [1]))):
                rc, codes, skipped = check(native, oracle, data, rt, flags, name, random.Random(rt), f"1,025 entries, {what}")
                assert rc == 0 and codes == {b"k": 1} and [s[0] for s in skipped] == [1]
        p = ld(2, b"".join(map_entry(b"s%05d" % i, C.fl(C.i64(i))) for i in range(1025)))
        assert _run(native, 1, flags, name, lambda inf, s: inf.update(pyref.frame_fast(p)))[0] == A.TFR_E_BATCH_TOO_LARGE


# --------------------------------------------------------------------------------------------
# 7. FAILFAST through tfr_infer_create_mode is tfr_infer_create
# --------------------------------------------------------------------------------------------
def _created(native, rt):
    h = native.C.c_void_p()
    native._check(native.lib().tfr_infer_create(rt, 0, native.C.byref(h)))
    inf = native.Infer.__new__(native.Infer)
    inf.h = h
    return inf


def _failfast(native, inf, feed):
    try:
        feed(inf)
        return 0, inf.result(), inf.skipped()
    except native.TfrError as e:
        return e.code, None, inf.skipped()
    finally:
        inf.close()


@pytest.mark.parametrize("rt", [0, 1])
def test_failfast_mode_is_the_old_create(native, rt):
    R = random.Random(30 + rt)
    for seed in range(48):
        b = C.batch(seed, rt, R.choice([1, 2, 33, 64, 200]))
        feed = lambda inf: inf.update(np.frombuffer(b.data, np.uint8))     # noqa: E731
        old = _failfast(native, _created(native, rt), feed)
        for flags in (0, A.TFR_F_VERIFY_CRC):
            assert _failfast(native, native.Infer(rt, 0, flags), feed) == old, f"seed {seed}: {b.describe()}"
        assert old[2] == []
        for make in (lambda: _created(native, rt), lambda: native.Infer(rt, 0, 0)):
            seed_r = random.Random(seed)
            assert _failfast(native, make(), lambda inf: _blocks(inf, b, seed_r))[:2] == old[:2]


# --------------------------------------------------------------------------------------------
# 8. PERMISSIVE's name
# --------------------------------------------------------------------------------------------
def test_the_corrupt_record_name_in_every_place_and_kind(native, oracle):
    R = random.Random(8)
    for rt in (0, 1):
        for m in ((0, 1) if rt == 1 else (0,)):
            for k in range(12):
                val = planted_value(random.Random(100 * m + k), m)
                for pad in (0, 40):
                    p = ld(m + 1, _fill(pad, b"p", m) + map_entry(CORRUPT, val) + _fill(pad, b"q", m)) + ld(1, map_entry(b"k", C.i64(1)))
                    data = framed([p, ld(1, map_entry(b"k", C.f32(1.0)))])
                    rc, codes, skipped = check(native, oracle, data, rt, PERM, CORRUPT, R, f"rt {rt} map {m} value {val.hex()}")
                    assert rc == 0 and CORRUPT not in codes and skipped == [] and codes[b"k"] == 2
                    rc2, codes2, skipped2 = check(native, oracle, data, rt, DROP, None, R, f"rt {rt} map {m} value {val.hex()}")
                    assert rc2 in (0, A.TFR_E_UNSUPPORTED_TYPE)
                    assert (CORRUPT in codes2) != bool(skipped2)             # an ordinary name: merged, or its record fails
    # a custom name is the one ignored; the default one is then ordinary
    p = ld(1, map_entry(b"bad", C.UNSET) + map_entry(CORRUPT, C.i64(1)))
    rc, codes, skipped = check(native, oracle, framed([p]), 0, PERM, b"bad", R, "custom name")
    assert (rc, codes, skipped) == (0, {CORRUPT: 1}, [])


# --------------------------------------------------------------------------------------------
# 9. io.DefaultSource.inferSchema
# --------------------------------------------------------------------------------------------
def _good(i):
    return ld(1, map_entry(b"a", C.i64(i)) + map_entry(b"b", C.f32(0.5 * i)) + map_entry(b"s", C.byt(b"v%d" % i)))


def _write(path, payloads, crc=()):
    data = framed(payloads, crc)
    with open(path, "wb") as f:
        f.write(data)
    return data


SCHEMA = [("a", LongType()), ("b", FloatType()), ("s", StringType())]


def _logged(caplog):
    return [r.getMessage() for r in caplog.records if "schema inference skipped" in r.getMessage()]


@pytest.mark.parametrize("block", [None, 64])
def test_infer_schema_modes(native, oracle, tmp_path, caplog, monkeypatch, block):
    if block:
        monkeypatch.setattr(tio.TFRecordFileReader, "BLOCK_BYTES", block)
    ps = [_good(i) for i in range(20)]
    ps[3] = ld(1, map_entry(b"a", C.UNSET) + map_entry(b"only_bad", C.i64(1)))
    ps[7] = ps[7] + b"\x0a\x05\x01"
    path = str(tmp_path / "part-00000.tfrecord")
    data = _write(path, ps, crc=[11])
    src = tio.DefaultSource()
    with pytest.raises(Exception):
        src.inferSchema({}, [path])                                              # FAILFAST
    with caplog.at_level(logging.WARNING):
        sch = src.inferSchema({"mode": "dropMalformed"}, [path])
    assert [(f.name, f.dataType) for f in sch] == SCHEMA
    off3 = sum(16 + len(p) for p in ps[:3])
    assert _logged(caplog) == [f"{path}: schema inference skipped 3 malformed record(s); the first at file offset {off3} (TFR_E_KIND_MISMATCH)"]
    caplog.clear()
    for opts, name in (({"mode": "PERMISSIVE"}, "_corrupt_record"), ({"mode": "permissive", "columnNameOfCorruptRecord": "bad"}, "bad")):
        with caplog.at_level(logging.WARNING):
            sch = src.inferSchema(opts, [path])
        assert [(f.name, f.dataType, f.nullable) for f in sch] == [(n, t, True) for n, t in SCHEMA] + [(name, BinaryType(), True)]
        assert len(_logged(caplog)) == 1
        caplog.clear()
        # the inferred schema reads the file back under the same options: PERMISSIVE's rows
        rows = src.load(path, sch, opts)
        e = P.expected(oracle, data, sch, 0, PERM, len(SCHEMA))
        assert rows == [tuple(c.get(r) for c in e.columns) for r in range(e.info["n_rows"])]
        assert len(rows) == 20 and rows[3][:3] == (None, None, None) and rows[3][3] == ps[3]


def test_infer_schema_passes_over_a_file_of_bad_records(native, tmp_path, caplog):
    d = tmp_path / "t"
    d.mkdir()
    bad, good = str(d / "part-00000.tfrecord"), str(d / "part-00001.tfrecord")
    _write(bad, [ld(1, map_entry(b"x", C.UNSET)) for _ in range(5)])
    _write(good, [_good(i) for i in range(4)])
    src = tio.DefaultSource()
    with caplog.at_level(logging.WARNING):
        sch = src.inferSchema({"mode": "DROPMALFORMED"}, [bad, good])
    assert [(f.name, f.dataType) for f in sch] == SCHEMA
    assert len(_logged(caplog)) == 1 and "skipped 5 malformed" in _logged(caplog)[0]
    sch = src.inferSchema({"mode": "PERMISSIVE"}, [bad, good])
    assert [f.name for f in sch] == ["a", "b", "s", "_corrupt_record"]
    sch = src.inferSchema({"mode": "PERMISSIVE"}, [bad])
    assert [(f.name, f.dataType) for f in sch] == [("_corrupt_record", BinaryType())]
    with pytest.raises(Exception):
        src.inferSchema({"mode": "FAILFAST"}, [bad, good])
