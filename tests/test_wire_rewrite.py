"""The wire rewriter (tests/wire_rewrite.py) and the C oracle, pinned on the CPU: the GPU wire-fuzz tests
(tests/test_gpu_wire_fuzz.py) compare the decoders with the oracle, so they are only as good as these two.

  * the canonical form is the reference writer's bytes (oracle writer, M/TFRecordSerializer.scala:20-60);
  * class A (equivalent rewrites): the oracle decodes every rewritten record to the source rows, bit for bit, and so
    does upb (google.protobuf) + pyref's restatement of TFRecordDeserializer wherever upb agrees with protobuf-java;
  * class B (errors with a valid CRC): the oracle reports the constructed status, row and field, with the source rows
    in front of the failing one;
  * class C (byte-wise damage, CRC recomputed): the oracle rejects a payload as malformed exactly when upb does, apart
    from the two listed upb deviations (a map entry with an unknown field, a tag longer than five bytes)."""
import random

import numpy as np
import pytest
from google.protobuf.message import DecodeError

import wire_rewrite as W
from oracle import pyref
from util import assert_columns_equal, slice_columns
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

SHAPES = [(1, 0, False), (12, 0, False), (13, 0, True), (65, 0, False), (129, 0, False),
          (13, 1, False), (40, 1, True)]                   # (width, record type, big records)


def _corpus(seed, width, rt, big, n):
    sch, gen = W.make_schema(seed, width, rt, big=big, with_2d=(rt == 0 and width == 12))
    r = np.random.default_rng(seed + 1)
    rows = [gen(r) for _ in range(n)]
    return sch, rows, W.source_columns(sch, rows, rt)


def _upb_rows(sch, payloads, rt):
    if rt == TFR_RT_SEQUENCE_EXAMPLE:
        return [pyref.deserialize_sequence_example(sch, pyref.SequenceExample.FromString(p)) for p in payloads]
    return [pyref.deserialize_example(sch, pyref.Example.FromString(p)) for p in payloads]


@pytest.mark.parametrize("width,rt,big", SHAPES)
def test_canonical_is_the_writers_bytes(oracle, width, rt, big):
    sch, rows, cols = _corpus(11 + width, width, rt, big, 40)
    if any(isinstance(f.dataType, NullType) for f in sch.fields):
        sch = StructType([f for f in sch.fields if not isinstance(f.dataType, NullType)])
        keep = [i for i, c in enumerate(cols) if c.elem_type != A.TFR_T_NULL]
        rows = [tuple(r[i] for i in keep) for r in rows]
        cols = [cols[i] for i in keep]
    want, rc, _ = oracle.encode(cols, sch, rt)
    assert rc == 0
    assert W.frame(W.canonical(sch, row, rt) for row in rows) == want


@pytest.mark.parametrize("cls", W.A_CLASSES)
@pytest.mark.parametrize("width,rt,big", SHAPES)
def test_equivalent_rewrites_decode_to_the_source_rows(oracle, cls, width, rt, big):
    n = 24
    for seed in range(3):
        sch, rows, cols = _corpus(1000 * seed + width, width, rt, big, n)
        R = random.Random(f"{cls}/{seed}/{width}/{rt}")
        out = [W.rewrite(sch, row, rt, cls, R, W=R.choice([12, 4])) for row in rows]
        payloads = [p for p, _ in out]
        what = f"class {cls}, seed {seed}, width {width}, record type {rt}"
        got = oracle.decode(W.frame(payloads), sch, rt)
        assert got.info["error_code"] == 0, (what, got.info, [w for _, w in out][got.info["error_row"]])
        assert_columns_equal(got.columns, cols, sch.names, what)
        # upb, wherever it agrees with protobuf-java (it keeps a map entry with an unknown field as an unknown field)
        for r, (p, how) in enumerate(out):
            if W.upb_deviation(p, rt):
                continue
            upb = W.source_columns(sch, _upb_rows(sch, [p], rt), rt)
            assert_columns_equal(upb, slice_columns(cols, r, r + 1), sch.names, f"{what}, row {r} ({how}) through upb: {p.hex()}")


def test_equivalent_rewrites_cover_every_variant():
    """each class draws from its variants at random: over the seeds the tests use, every variant occurs"""
    sch, rows, _ = _corpus(7, 40, 1, False, 200)
    seen = set()
    for cls in W.A_CLASSES:
        R = random.Random(cls)
        for row in rows:
            seen.add((cls, W.rewrite(sch, row, 1, cls, R)[1].split(" in ")[0].split(" at ")[0].split(" (")[0]))
    for what in ("reversed", "shuffled", "rot1", "rot5", "unpacked list", "mixed list", "packed_segments list",
                 "value before key", "key twice, decoy first,", "feature_lists before context", "empty context / feature_lists omitted"):
        assert any(w.startswith(what.split(" list")[0]) for _, w in seen), (what, sorted(seen))
    extra = {w.split(" (")[0] for c, w in seen if c == "extra"}
    assert {f"extra key {v}" for v in W.EXTRA_KEYS} <= extra, extra


def test_fnv_collision_and_slot_keys():
    a, b = W.fnv_collision()
    assert a != b and len(a) == len(b) == 8 and W.fnv1a(a) == W.fnv1a(b)
    sch, _ = W.make_schema(3, 65)
    assert a.decode() in sch.names
    R = random.Random(1)
    k = W._extra_key(R, sch, "slot")
    names = {f.encode() for f in sch.names}
    m = W.ht_mask(len(sch.fields))
    assert k not in names and any(W.fnv1a(k) & m == W.fnv1a(x) & m and W.fnv1a(k) != W.fnv1a(x) for x in names)
    assert W._extra_key(R, sch, "fnv") == b


ERROR_ROWS = [0, 31, 32, 20, 47]


@pytest.mark.parametrize("cls", W.B_CLASSES)
@pytest.mark.parametrize("width,rt,big", SHAPES)
def test_error_rewrites_report_the_constructed_status(oracle, cls, width, rt, big):
    n = 48
    sch, rows, cols = _corpus(77 + width, width, rt, big, n)
    R = random.Random(f"{cls}/{width}/{rt}")
    tried = 0
    for er in ERROR_ROWS:
        e = W.error_record(sch, rows[er], rt, cls, R)
        if e is None:
            continue
        tried += 1
        p, code, field, how = e
        payloads = [W.canonical(sch, row, rt) for row in rows]
        payloads[er] = p
        got = oracle.decode(W.frame(payloads), sch, rt)
        what = f"{cls} ({how}) at row {er}: {p.hex()}"
        if code == 0:
            assert got.info["error_code"] == 0, (what, got.info)
            assert_columns_equal(got.columns, cols, sch.names, what)
            continue
        assert (got.info["error_code"], got.info["error_row"], got.info["error_field"], got.info["n_rows"]) == (code, er, field, er), (what, got.info)
        assert_columns_equal(got.columns, slice_columns(cols, 0, er), sch.names, what)
    if cls in ("kind_mismatch", "kind_not_set", "malformed", "groups_24", "groups_25", "empty_scalar", "null_in_nonnull") \
            or (cls == "bad_nesting" and (rt == 1 or width == 12)):
        assert tried, "schema cannot express this error"


@pytest.mark.parametrize("width,rt,big", SHAPES)
def test_two_errors_the_first_wins(oracle, width, rt, big):
    """two failing rows in one batch: the first row's error; two failing fields in one record (the later field's entry
    first on the wire): the first field in schema order"""
    sch, rows, cols = _corpus(5 + width, width, rt, big, 48)
    R = random.Random(width)
    payloads = [W.canonical(sch, row, rt) for row in rows]
    p1, c1, f1, _ = W.error_record(sch, rows[31], rt, "kind_not_set", R)
    p2, c2, f2, _ = W.error_record(sch, rows[32], rt, "malformed", R)
    payloads[31], payloads[32] = p1, p2
    got = oracle.decode(W.frame(payloads), sch, rt)
    assert (got.info["error_code"], got.info["error_row"], got.info["error_field"]) == (c1, 31, f1)
    two = W.two_errors_in_one_record(sch, rows[20], rt, R)
    if two is None:
        return
    p, code, field, how = two
    payloads = [W.canonical(sch, row, rt) for row in rows]
    payloads[20] = p
    got = oracle.decode(W.frame(payloads), sch, rt)
    assert (got.info["error_code"], got.info["error_row"], got.info["error_field"]) == (code, 20, field), how


def test_nested_groups_are_skipped_by_the_oracle_and_upb(oracle):
    """groups nested 24 and 25 deep: protobuf-java skips both, and so do the oracle and upb (the GPU parsers' 24-deep
    group stack is the documented deviation, checked in test_gpu_wire_fuzz.py)"""
    sch, rows, cols = _corpus(3, 12, 0, False, 1)
    for d in (24, 25):
        p, code, field, _ = W.error_record(sch, rows[0], 0, f"groups_{d}", random.Random(0))
        assert code == 0
        got = oracle.decode(W.frame([p]), sch)
        assert got.info["error_code"] == 0
        assert_columns_equal(got.columns, cols, sch.names, f"groups {d}")
        pyref.Example.FromString(p)


@pytest.mark.parametrize("rt", [0, 1])
def test_damaged_payloads_oracle_rejects_exactly_what_upb_rejects(oracle, rt):
    """byte-wise damage (flip, insert, delete, overwrite) of one payload, CRC recomputed: the oracle's
    MALFORMED_PROTO is upb's DecodeError, on every payload.  The listed exceptions (upb_deviation) are upb's handling of
    map entries that carry an unknown field and of tags longer than five bytes: such a payload must really have one, and
    it is counted, not dropped."""
    sch, rows, _ = _corpus(99 + rt, 13, rt, False, 60)
    R = random.Random(rt)
    cls_of = pyref.SequenceExample if rt else pyref.Example
    agree = deviations = 0
    for t in range(2500):
        row = rows[t % len(rows)]
        base = W.canonical(sch, row, rt) if t % 3 else W.rewrite(sch, row, rt, R.choice(W.A_CLASSES), R)[0]
        p, how = W.mutate(base, R)
        got = oracle.decode(W.frame([p]), sch, rt, copy_columns=False)
        o_bad = got.info["error_code"] == A.TFR_E_MALFORMED_PROTO
        try:
            cls_of.FromString(p)
            u_bad = False
        except DecodeError:
            u_bad = True
        if o_bad == u_bad:
            agree += 1
            continue
        # each deviation goes one way only: upb never looks inside a map entry it keeps as an unknown field (so it can
        # only accept what protobuf-java rejects), and a long tag can only make upb reject what protobuf-java accepts
        dev = W.upb_deviation(p, rt)
        expected = {"unknown field inside a map entry": (True, False), "tag longer than five bytes": (False, True)}
        assert expected.get(dev) == (o_bad, u_bad), (how, o_bad, u_bad, dev, p.hex())
        deviations += 1
    assert agree >= 2400, (agree, deviations)
