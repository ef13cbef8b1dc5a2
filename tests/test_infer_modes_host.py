"""Schema inference in DROPMALFORMED and PERMISSIVE, pinned on the CPU (no GPU): tests/test_gpu_infer_modes.py compares the
GPU with `infer_modes_oracle.infer_mode`, so it is only as good as these.

  * over tests/infer_corpus.py's seeded batches of every MODES entry, for both record types, the tolerant
    inference is test_infer_corpus's restatement of TensorFlowInferSchema over upb applied to the records that pass
    (CRC, parse, value errors), and its skipped list is exactly the records that do not; the corrupt-record column's
    name is planted in some records, ignored in PERMISSIVE and an ordinary name in DROPMALFORMED;
  * FAILFAST through the new entry point is the old one;
  * `inferSchema` refuses an unknown `mode` before it opens a file, tfr_infer_create_mode refuses bad arguments before
    any device work, and the new symbols are declared, bound, exported and reachable from the JNI shim."""
import os
import random
import re
import subprocess

import pytest

import infer_corpus as C
import infer_modes_oracle as M
from oracle import pyref
from oracle.pyref import ld, map_entry
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from test_infer_corpus import _deviates, _parses, _restated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROP = A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED
PERM = A.TFR_F_DEFAULT | A.TFR_F_PERMISSIVE
CORRUPT = b"_corrupt_record"


def planted_value(R: random.Random, m: int) -> bytes:
    """a value for the corrupt-record column's name in map m: every kind, kind not set, and in feature_lists an empty
    FeatureList, a step whose kind is not set and all-empty steps"""
    if m == 0:
        return R.choice([C.i64(1), C.i64(1, 2), C.f32(1.5), C.byt(b"x"), C.i64(), C.byt(), C.UNSET])
    return R.choice([C.fl(C.i64(1)), C.fl(C.f32(1.0, 2.0)), C.fl(C.byt(b"s")), b"", C.fl(C.UNSET),
                     C.fl(C.i64(1), C.UNSET), C.fl(C.i64(), C.f32())])


def plant(R: random.Random, rt: int, payload: bytes, name: bytes = CORRUPT) -> bytes:
    """`payload` with an entry keyed `name` put in front (a repeated top-level field merges, so the record is the same
    record plus that entry, and a record that does not parse still does not)"""
    m = R.randrange(2) if rt == 1 else 0
    return ld(m + 1, map_entry(name, planted_value(R, m)))[:] + payload


def framed(payloads, crc_rows=(), lencrc_row=None, truncated=False) -> bytes:
    frames = [pyref.frame_fast(p) for p in payloads]
    for r in crc_rows:
        f = bytearray(frames[r])
        f[-1 - (r % 4)] ^= 0x10                                    # the stored data CRC no longer matches
        frames[r] = bytes(f)
    if lencrc_row is not None:
        f = bytearray(frames[lencrc_row])
        f[8] ^= 0x01                                               # the stored length CRC no longer matches
        frames[lencrc_row] = bytes(f)
    if truncated and frames:
        frames[-1] = frames[-1][:12 + (len(frames[-1]) - 12) // 2]
    return b"".join(frames)


def _passes(p: bytes, rt: int) -> bool:
    """the record's verdict under TensorFlowInferSchema over upb (a conflict inside one record is no record error)"""
    return _parses(p, rt) and _restated([p], rt)[0] in (0, A.TFR_E_UNSUPPORTED_TYPE)


def corpus(seed: int, rt: int, mode: str):
    """(original payloads, planted payloads, data CRC flipped rows, final frame truncated) of one seeded batch; records
    where upb deviates from protobuf-java are left out"""
    b = C.batch(seed, rt, 40, mode=mode)
    R = random.Random(f"modes/{seed}/{rt}/{mode}")
    keep = [row for row in range(len(b.payloads)) if not _deviates(b, row)]
    orig = [b.payloads[row] for row in keep]
    planted = [plant(R, rt, p) if R.random() < 0.3 else p for p in orig]
    crc = {keep.index(b.crc_row)} if b.crc_row in keep else set()
    if R.random() < 0.3 and orig:
        crc.add(R.randrange(len(orig)))
    return orig, planted, sorted(crc), b.truncated


@pytest.mark.parametrize("rt", [0, 1])
@pytest.mark.parametrize("mode", sorted(set(C.MODES)))
def test_oracle_is_the_restated_inference_of_the_kept_records(oracle, rt, mode):
    seen = {}
    for seed in range(12):
        orig, planted, crc, truncated = corpus(seed, rt, mode)
        data = framed(planted, crc, truncated=truncated)
        n = len(planted) - (1 if truncated else 0)             # the truncated frame is no record
        ends = [0]
        for p in planted:
            ends.append(ends[-1] + 16 + len(p))
        for flags, name, judged in ((PERM, CORRUPT, orig), (DROP, None, planted)):
            kept = [judged[r] for r in range(n) if r not in crc and _passes(judged[r], rt)]
            want_rc, want_codes = _restated(kept, rt)
            want_skipped = [r for r in range(n) if r in crc or not _passes(judged[r], rt)]
            rc, codes, skipped = M.infer_mode(data, rt, flags, name)
            what = f"seed {seed}, {'PERMISSIVE' if name else 'DROPMALFORMED'}"
            assert [r for r, _, _ in skipped] == want_skipped, what
            assert all(off == ends[r] for r, off, _ in skipped), what
            assert all(code == A.TFR_E_CRC_DATA for r, _, code in skipped if r in crc), what
            assert all(code in (A.TFR_E_MALFORMED_PROTO, A.TFR_E_KIND_MISMATCH, A.TFR_E_EMPTY_SCALAR)
                       for r, _, code in skipped if r not in crc), what
            if truncated:
                assert rc == A.TFR_E_TRUNCATED, what
                if want_rc == 0:
                    assert codes == want_codes, what
            else:
                assert (rc, codes if rc == 0 else None) == (want_rc, want_codes), what
            seen[rc] = seen.get(rc, 0) + 1
            if name:
                assert CORRUPT not in codes, what
    assert seen, seen


def test_planted_name_is_an_ordinary_feature_without_permissive(oracle):
    p = ld(1, map_entry(CORRUPT, C.i64(1, 2)) + map_entry(b"a", C.f32(1.0)))
    assert M.infer_mode(framed([p]), 0, DROP) == (0, {CORRUPT: 4, b"a": 2}, [])
    assert M.infer_mode(framed([p]), 0, PERM, CORRUPT) == (0, {b"a": 2}, [])
    bad = ld(1, map_entry(CORRUPT, C.UNSET) + map_entry(b"a", C.f32(1.0)))
    assert M.infer_mode(framed([bad]), 0, DROP) == (0, {}, [(0, 0, A.TFR_E_KIND_MISMATCH)])
    assert M.infer_mode(framed([bad]), 0, PERM, CORRUPT) == (0, {b"a": 2}, [])


@pytest.mark.parametrize("rt", [0, 1])
def test_failfast_entry_point_is_the_old_one(oracle, rt):
    for seed in range(24):
        b = C.batch(seed, rt, 30)
        rc, codes = oracle.infer(b.data, rt)
        assert M.infer_mode(b.data, rt, 0) == (rc, codes, [])
        assert M.infer_mode(b.data, rt, A.TFR_F_DEFAULT) == (rc, codes, [])


def test_framing_errors_end_the_call_with_what_came_before(oracle):
    ps = [ld(1, map_entry(b"k%d" % i, C.i64(i))) for i in range(5)]
    ps[1] = ld(1, map_entry(b"bad", C.UNSET))
    assert M.infer_mode(framed(ps, lencrc_row=3), 0, DROP) == (
        A.TFR_E_CRC_LENGTH, {b"k0": 1, b"k2": 1}, [(1, 16 + len(ps[0]), A.TFR_E_KIND_MISMATCH)])
    rc, codes, skipped = M.infer_mode(framed(ps, truncated=True), 0, DROP)
    assert (rc, codes, [r for r, _, _ in skipped]) == (A.TFR_E_TRUNCATED, {b"k0": 1, b"k2": 1, b"k3": 1}, [1])


# --------------------------------------------------------------------------------------------
# the public surface, without a device
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["LENIENT", "", "drop", "FAIL_FAST"])
def test_infer_schema_refuses_an_unknown_mode_before_opening_a_file(mode):
    with pytest.raises(_native.IllegalArgumentException, match=f"mode {mode}"):
        tio.DefaultSource().inferSchema({"mode": mode}, ["/nonexistent/part-00000.tfrecord"])


def test_infer_schema_byte_array_is_fixed_in_every_mode(tmp_path):
    for mode in ("FAILFAST", "dropmalformed", "Permissive"):
        sch = tio.DefaultSource().inferSchema({"mode": mode, "recordType": "ByteArray"}, [str(tmp_path / "absent")])
        assert [f.name for f in sch] == ["byteArray"]


@pytest.mark.parametrize("rt, flags, name, what", [
    (0, PERM | A.TFR_F_DROP_MALFORMED, CORRUPT, "exclude each other"),
    (0, 0x8, None, "unknown flag"),
    (0, A.TFR_F_DEFAULT | 0x100, None, "unknown flag"),
    (0, DROP, CORRUPT, "needs TFR_F_PERMISSIVE"),
    (0, A.TFR_F_DEFAULT, CORRUPT, "needs TFR_F_PERMISSIVE"),
    (1, PERM, None, "corrupt-record column's name"),
    (1, PERM, b"", "corrupt-record column's name"),
])
def test_create_mode_refuses_before_device_work(rt, flags, name, what):
    L = _native.lib()
    out = _native.C.c_void_p()
    rc = L.tfr_infer_create_mode(rt, 0, flags, name, len(name) if name is not None else 0, _native.C.byref(out))
    assert rc == A.TFR_E_INVALID_ARG and not out.value
    assert what in L.tfr_last_error().decode()


def test_create_mode_name_length_and_record_type():
    L = _native.lib()
    out = _native.C.c_void_p()
    assert L.tfr_infer_create_mode(0, 0, PERM, b"x", 1 << 24, _native.C.byref(out)) == A.TFR_E_INVALID_ARG
    assert L.tfr_infer_create_mode(0, 0, PERM, b"x", -1, _native.C.byref(out)) == A.TFR_E_INVALID_ARG
    assert L.tfr_infer_create_mode(0, 0, DROP, None, 1, _native.C.byref(out)) == A.TFR_E_INVALID_ARG
    assert L.tfr_infer_create_mode(0, 0, DROP, None, 0, None) == A.TFR_E_INVALID_ARG
    assert L.tfr_infer_create_mode(2, 0, DROP, None, 0, _native.C.byref(out)) == A.TFR_E_BAD_RECORD_TYPE
    assert not out.value
    with pytest.raises(_native.IllegalArgumentException):
        _native.Infer(2, 0, DROP)
    with pytest.raises(_native.TfrError, match="exclude each other"):
        _native.Infer(0, 0, PERM | A.TFR_F_DROP_MALFORMED, "_corrupt_record")


def test_new_symbols_are_declared_bound_and_exported():
    hdr = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    assert re.search(r"int32_t\s+tfr_infer_create_mode\(int32_t record_type,\s*int32_t device,\s*uint32_t flags,\s*"
                     r"const char\* corrupt_name,\s*int32_t corrupt_name_len,\s*tfr_infer\*\* out\);", hdr)
    assert re.search(r"int32_t\s+tfr_infer_skipped\(tfr_infer\*,\s*int64_t\* n_skipped,\s*int64_t\* record,\s*"
                     r"int64_t\* offset,\s*int32_t\* code,\s*int64_t cap\);", hdr)
    L = _native.lib()
    for s in ("tfr_infer_create_mode", "tfr_infer_skipped"):
        assert s in _native.EXPORTS and hasattr(L, s)
    out = _native.C.c_int64()
    assert L.tfr_infer_skipped(None, _native.C.byref(out), None, None, None, 0) == A.TFR_E_INVALID_ARG


def test_jni_shim_has_the_mode_entry_points():
    src = os.path.join(ROOT, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    text = open(src).read()
    for sym in ("TfrGpu_inferCreateMode", "TfrGpu_inferSkipped"):
        assert "Java_com_linkedin_spark_datasources_tfrecord_" + sym in text
    assert "tfr_infer_create_mode(" in text and "tfr_infer_skipped(" in text
    p = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-DTFR_BUILD_JNI", "-I", os.path.join(ROOT, "tests", "jni_stub"),
                        "-I", os.path.join(ROOT, "include"), src], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
