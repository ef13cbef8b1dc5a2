"""tests/infer_corpus.py and the oracle's inference, pinned on the CPU: tests/test_gpu_infer_fuzz.py compares the GPU with
`oracle.infer`, so it is only as good as these.

  * the hand-written regressions give the verdicts TensorFlowInferSchema gives them;
  * every generated record parses or fails under google.protobuf (upb) exactly as the oracle's parse says (apart from
    upb's one deviation: a map entry with an unknown field);
  * where the records parse, the oracle's result is a short restatement of TensorFlowInferSchema over the upb messages,
    with each map in the order of the first wire occurrence of its keys;
  * the generator is deterministic for a seed."""
import pytest
from google.protobuf.message import DecodeError

import infer_corpus as C
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A


def test_the_colliding_names_share_their_hash():
    assert C.COLL_A != C.COLL_B and C.fnv1a64(C.COLL_A) == C.fnv1a64(C.COLL_B)
    assert len(C.COLL_A) == len(C.COLL_B) == 16


@pytest.mark.parametrize("name,payload,rt,rc,codes", C.payload_table(), ids=[t[0] for t in C.payload_table()])
def test_regressions_oracle_verdicts(oracle, name, payload, rt, rc, codes):
    got_rc, got = oracle.infer(pyref.frame(payload), rt)
    assert got_rc == rc
    if rc == 0:
        assert got == codes
    assert _restated([payload], rt) == (rc, codes) if rc != A.TFR_E_MALFORMED_PROTO else _parses(payload, rt) is False


# --------------------------------------------------------------------------------------------
# TensorFlowInferSchema over upb
# --------------------------------------------------------------------------------------------
def _varint(b, p):
    v = s = 0
    while True:
        c = b[p]; p += 1
        v |= (c & 0x7F) << s; s += 7
        if c < 0x80:
            return v, p


def _walk(b):
    """(field number, wire type, payload of a length-delimited field) of a well-formed message; groups skipped whole"""
    p, out, depth = 0, [], 0
    while p < len(b):
        t, p = _varint(b, p)
        f, w = t >> 3, t & 7
        if w == 2:
            n, p = _varint(b, p)
            if not depth:
                out.append((f, w, b[p:p + n]))
            p += n
        elif w == 0:
            _, p = _varint(b, p)
        elif w in (1, 5):
            p += 8 if w == 1 else 4
        elif w == 3:
            depth += 1
        elif w == 4:
            depth -= 1
    return out


def _key_order(payload, rt, field):
    """keys of map `field` (1: features / context, 2: feature_lists) in the order of their first wire occurrence"""
    order = {}
    for f, w, body in _walk(payload):
        if w != 2 or f != field or (f == 2 and rt != 1):
            continue
        for f2, w2, ent in _walk(body):
            if (f2, w2) != (1, 2):
                continue
            key = b""
            for f3, w3, v in _walk(ent):
                if (f3, w3) == (1, 2):
                    key = v
            order.setdefault(key, None)
    return list(order)


def _code(feat):
    """inferField + parse*List (M/TensorFlowInferSchema.scala:132-188); None: the kind is not set"""
    kind = feat.WhichOneof("kind")
    if kind is None:
        return None
    n = len(getattr(feat, kind).value)
    base = {"int64_list": 1, "float_list": 2, "bytes_list": 3}[kind]
    return 0 if n == 0 else base + 3 if n > 1 else base


def _parses(payload, rt):
    try:
        (pyref.SequenceExample if rt == 1 else pyref.Example).FromString(payload)
        return True
    except DecodeError:
        return False


def _restated(payloads, rt):
    """-> (status, names -> codes) of TensorFlowInferSchema over upb's parse of each payload"""
    merged, conflict = {}, False

    def merge(k, c):
        nonlocal conflict
        old = merged.get(k)
        if old is not None and old != c and 0 not in (old, c) and 10 in (old, c):
            conflict = True                                         # getNumericPrecedence(ArrayType(ArrayType(null)))
        merged[k] = c if old is None else max(old, c)

    for p in payloads:
        msg = (pyref.SequenceExample if rt == 1 else pyref.Example).FromString(p)
        fmap = msg.context.feature if rt == 1 else msg.features.feature
        for k in _key_order(p, rt, 1):
            c = _code(fmap[k.decode()])
            if c is None:
                return A.TFR_E_KIND_MISMATCH, None
            merge(k, c)
        if rt != 1:
            continue
        for k in _key_order(p, rt, 2):
            steps = msg.feature_lists.feature_list[k.decode()].feature
            if not steps:
                return A.TFR_E_EMPTY_SCALAR, None                   # empty.reduceLeft
            cs = [_code(s) for s in steps]
            if None in cs:
                return A.TFR_E_KIND_MISMATCH, None
            c = max(cs)
            merge(k, 10 if c == 0 else 7 + (c - 1) % 3)
    return (A.TFR_E_UNSUPPORTED_TYPE, None) if conflict else (0, merged)


def _deviates(b, row):
    return any(r == row and C.UPB_DEVIATES in n for r, n in b.notes)


@pytest.mark.parametrize("rt", [0, 1])
def test_records_parse_under_upb_as_under_the_oracle(oracle, rt):
    checked = failed = 0
    for seed in range(60):
        b = C.batch(seed, rt, 30)
        for row, p in enumerate(b.payloads):
            if _deviates(b, row):
                continue
            mal = oracle.infer(pyref.frame_fast(p), rt)[0] == A.TFR_E_MALFORMED_PROTO
            assert _parses(p, rt) == (not mal), f"seed {seed} row {row}: oracle malformed {mal}; {b.describe()}; {p.hex()}"
            checked += 1
            failed += mal
    assert checked > 1000 and failed >= 5, (checked, failed)


@pytest.mark.parametrize("rt", [0, 1])
def test_oracle_is_the_restated_inference(oracle, rt):
    verdicts = {}
    for seed in range(60):
        b = C.batch(seed, rt, 40)
        keep = [p for row, p in enumerate(b.payloads) if not _deviates(b, row) and _parses(p, rt)]
        rc, codes = oracle.infer(b"".join(pyref.frame_fast(p) for p in keep), rt)
        want = _restated(keep, rt)
        assert (rc, codes if rc == 0 else None) == want, f"seed {seed}: {b.describe()}"
        verdicts[rc] = verdicts.get(rc, 0) + 1
    expect = {0, A.TFR_E_KIND_MISMATCH} | ({A.TFR_E_EMPTY_SCALAR, A.TFR_E_UNSUPPORTED_TYPE} if rt == 1 else set())
    assert expect <= set(verdicts), verdicts


def test_the_generator_is_deterministic():
    for seed in range(8):
        for rt in (0, 1):
            a, b = C.batch(seed, rt, 25), C.batch(seed, rt, 25)
            assert a.data == b.data and a.notes == b.notes and a.frame_ends == b.frame_ends
    assert C.batch(1, 0, 25).data != C.batch(2, 0, 25).data


def test_the_generator_covers_its_shapes():
    """names of every kind, duplicate keys at every distance, errors in every place, every framing damage"""
    notes, modes = [], set()
    for seed in range(80):
        for rt in (0, 1):
            b = C.batch(seed, rt, 40)
            notes += [n for _, n in b.notes]
            modes.add((b.crc_row is not None, b.truncated))
    text = " | ".join(notes)
    for d in (0, 31, 32, 33, 70):
        assert f"at distance {d}" in text
    for kind in C.VALUE_ERRORS:
        for place in C.PLACES:
            assert f"{kind} {place}" in text, (kind, place)
    for kind in C.MALFORMED:
        for m in (0, 1):
            assert any(f"{kind} in {w} of map {m}" in text for w in ("map", "top", "value")), kind
    assert {(True, False), (False, True), (False, False)} <= modes
