"""CPU tests of TFR_F_RESYNC: the sequential walker (resync_walk.py) pinned clause by clause on hand-built bytes and by a
property test over block cuts, the flag's argument checks, the resyncFraming option, the header, the bindings and the JNI
shim.  The GPU against the walker: test_gpu_resync.py."""
import os
import random
import re
import struct
import subprocess

import pytest

import resync_walk as RW
from oracle.pyref import frame, masked_crc32c
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import BinaryType, LongType, StructField, StructType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CRC_LEN, TRUNC, TOO_LARGE = A.TFR_E_CRC_LENGTH, A.TFR_E_TRUNCATED, A.TFR_E_RECORD_TOO_LARGE


def hdr(length, ok=True):
    h = struct.pack("<Q", length)
    return h + struct.pack("<I", masked_crc32c(h) ^ (0 if ok else 1))


def recs(*sizes):
    return [frame(bytes([i + 1]) * n) for i, n in enumerate(sizes)]


def spans(entries):
    return [(e[0][0], e[1], e[2]) + e[3:] for e in entries]


F = recs(5, 9, 3, 20)
OFF = [0]
for f in F:
    OFF.append(OFF[-1] + len(f))


def test_clean_block_is_the_plain_chain():
    data = b"".join(F)
    assert RW.walk(data, True) == ([("frame", OFF[i], OFF[i + 1]) for i in range(4)], len(data))


@pytest.mark.parametrize("stray", range(1, 8))
def test_stray_bytes_stay_clean(stray):
    data = b"".join(F) + b"\x07" * stray
    ents, used = RW.walk(data, True)
    assert all(e[0] == "frame" for e in ents) and used == len(data)
    assert RW.walk(data, False) == (ents, OFF[4])


def test_bad_length_crc_resyncs_on_the_next_frame():
    bad = bytearray(F[1]); bad[9] ^= 4
    data = F[0] + bytes(bad) + F[2] + F[3]
    ents, used = RW.walk(data, True)
    assert ents == [("frame", 0, OFF[1]), ("region", OFF[1], OFF[2], CRC_LEN), ("frame", OFF[2], OFF[3]), ("frame", OFF[3], OFF[4])]
    assert used == len(data)


def test_oversize_length_with_a_valid_crc():
    data = F[0] + hdr(1 << 31) + F[1][12:] + F[2]
    ents, _ = RW.walk(data, True)
    assert ents[1] == ("region", OFF[1], OFF[2], TOO_LARGE) and ents[2][0] == "frame"


@pytest.mark.parametrize("left", [8, 11])
def test_partial_header_at_eof(left):
    data = b"".join(F[:2]) + F[2][:left]
    assert RW.walk(data, True) == ([("frame", 0, OFF[1]), ("frame", OFF[1], OFF[2]), ("region", OFF[2], len(data), TRUNC)], len(data))
    assert RW.walk(data, False)[1] == OFF[2]                   # not final: the ordinary carry


def test_frame_past_eof():
    data = b"".join(F[:2]) + F[3][:-3]
    ents, used = RW.walk(data, True)
    assert ents[-1] == ("region", OFF[2], len(data), TRUNC) and used == len(data)
    assert RW.walk(data, False)[1] == OFF[2]


def test_undecided_incomplete_header():
    """not final: a garbage tail shorter than a header could still hold one"""
    bad = bytearray(F[0]); bad[8] ^= 1
    data = bytes(bad) + b"\x00\x01\x02"
    assert RW.walk(data, False) == ([], 0)
    ents, used = RW.walk(data, True)
    assert ents == [("region", 0, len(data), CRC_LEN)] and used == len(data)


def test_undecided_frame_past_end():
    """not final: a verified header whose frame runs past the block, before any resync point"""
    bad = bytearray(F[0]); bad[8] ^= 1
    data = bytes(bad) + b"zz" + F[3][:20]
    assert RW.walk(data, False) == ([], 0)
    # with the rest of that frame the region resolves there
    data2 = bytes(bad) + b"zz" + F[3]
    assert RW.walk(data2, False)[0] == [("region", 0, len(F[0]) + 2, CRC_LEN), ("frame", len(F[0]) + 2, len(data2))]


def test_horizon():
    """a resync point must end within H of o; beyond it a position is never decisive"""
    bad = bytearray(F[0]); bad[8] ^= 1
    data = bytes(bad) + b"\xff" * 40 + F[1]
    p = len(F[0]) + 40
    assert RW.walk(data, True, H=len(data))[0] == [("region", 0, p, CRC_LEN), ("frame", p, len(data))]
    assert RW.walk(data, True, H=len(data) - 1)[0] == [("region", 0, len(data), CRC_LEN)]
    assert RW.walk(data, False, H=len(data) - 1) == ([], 0)     # not final, no resync point within H: unresolved


def test_decoy_with_bad_payload_crc_is_skipped():
    body = b"decoy!!!"
    decoy = hdr(len(body)) + body + struct.pack("<I", masked_crc32c(body) ^ 1)
    bad = bytearray(F[0]); bad[8] ^= 1
    data = bytes(bad) + b"\x11" * 3 + decoy + b"\x22" * 5 + F[1]
    p = len(data) - len(F[1])
    assert RW.walk(data, True)[0] == [("region", 0, p, CRC_LEN), ("frame", p, len(data))]


def test_valid_frame_inside_garbage_is_where_resync_lands():
    bad = bytearray(F[0]); bad[8] ^= 1
    data = bytes(bad) + b"\x33" * 7 + F[2] + b"\x44" * 9 + F[1]
    p = len(F[0]) + 7
    ents, _ = RW.walk(data, True)
    assert ents[:2] == [("region", 0, p, CRC_LEN), ("frame", p, p + len(F[2]))]
    assert ents[2] == ("region", p + len(F[2]), p + len(F[2]) + 9, CRC_LEN)


def test_region_at_offset_zero_and_two_adjacent_regions():
    b0 = bytearray(F[0]); b0[8] ^= 1
    b1 = bytearray(F[1]); b1[9] ^= 1
    data = bytes(b0) + hdr(1 << 40) + b"\x00" * 4 + bytes(b1) + F[2]
    ents, _ = RW.walk(data, True)
    # the region of b0 ends where a frame verifies: the oversize header and b1 belong to it
    assert ents == [("region", 0, OFF[0] + len(data) - len(F[2]), CRC_LEN), ("frame", len(data) - len(F[2]), len(data))]
    # a frame-sized gap closes the first region only at a verified frame; two framing stops in a row give two regions
    data = bytes(b0) + F[3] + hdr(1 << 33) + F[1][12:] + F[2]
    ents, _ = RW.walk(data, True)
    kinds = [e[0] for e in ents]
    assert kinds == ["region", "frame", "region", "frame"] and ents[2][3] == TOO_LARGE


def _damaged(seed):
    R = random.Random(seed)
    fr = [frame(R.randbytes(R.randrange(0, 120))) for _ in range(60)]
    for _ in range(4):
        i = R.randrange(len(fr))
        k = R.randrange(4)
        f = bytearray(fr[i])
        if k == 0:
            f[8 + R.randrange(4)] ^= 1 << R.randrange(8)
        elif k == 1:
            f = bytearray(hdr((1 << 31) + 5) + bytes(f[12:]))
        elif k == 2:
            f = bytearray(R.randbytes(R.randrange(1, 40))) + f
        else:
            f = f[:R.randrange(1, len(f))]
        fr[i] = bytes(f)
    return b"".join(fr)


@pytest.mark.parametrize("seed", range(12))
def test_block_cuts_do_not_change_the_result(seed):
    """a damaged corpus walked in random block cuts, with carry, gives the entries of one whole-file walk (file offsets)"""
    data = _damaged(seed)
    whole, used = RW.walk(data, True)
    assert used == len(data)
    R = random.Random(1000 + seed)
    for _ in range(6):
        cuts = sorted(R.sample(range(1, len(data)), R.randrange(1, 12)))
        assert RW.walk_blocks(data, cuts) == whole, cuts
    H = 600                                                     # a small horizon: no damaged run here comes close to it
    whole_h, _ = RW.walk(data, True, H)
    cuts = list(range(H // 2, len(data), H // 2))
    assert RW.walk_blocks(data, cuts, H) == whole_h


# ---------------------------------------------------------------------------------------------
# flags and options
# ---------------------------------------------------------------------------------------------
DATA = StructType([StructField("a", LongType()), StructField("_corrupt_record", BinaryType())])
R_ = A.TFR_F_RESYNC


@pytest.mark.parametrize("flags", [R_, A.TFR_F_DEFAULT | R_, A.TFR_F_DROP_MALFORMED | R_, A.TFR_F_PERMISSIVE | R_])
def test_decoder_flag_combinations_are_refused(flags):
    S = _native.Schema(DATA, 0)
    out = _native.C.c_void_p()
    assert _native.lib().tfr_decoder_create(S.h, 0, flags, _native.C.byref(out)) == A.TFR_E_INVALID_ARG and not out.value
    assert "TFR_F_RESYNC" in _native.lib().tfr_last_error().decode()
    if flags & A.TFR_F_PERMISSIVE:
        assert _native.lib().tfr_decoder_create_permissive(S.h, 0, flags, 1, _native.C.byref(out)) == A.TFR_E_INVALID_ARG


@pytest.mark.parametrize("flags", [R_, A.TFR_F_DEFAULT | R_, A.TFR_F_DROP_MALFORMED | R_])
def test_infer_flag_combinations_are_refused(flags):
    out = _native.C.c_void_p()
    assert _native.lib().tfr_infer_create_mode(0, 0, flags, None, 0, _native.C.byref(out)) == A.TFR_E_INVALID_ARG and not out.value


@pytest.mark.parametrize("mode, value, flags", [
    ("DROPMALFORMED", "true", A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED | R_),
    ("DROPMALFORMED", "True", A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED | R_),
    ("DROPMALFORMED", "false", A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED),
    ("PERMISSIVE", "TRUE", A.TFR_F_DEFAULT | A.TFR_F_PERMISSIVE | R_),
    ("FAILFAST", "false", A.TFR_F_DEFAULT),
])
def test_resync_framing_option(mode, value, flags):
    assert tio._decoder_flags({"mode": mode, "resyncFraming": value}, DATA) == flags


@pytest.mark.parametrize("opts", [{"resyncFraming": "true"}, {"mode": "FAILFAST", "resyncFraming": "true"},
                                  {"mode": "DROPMALFORMED", "resyncFraming": "yes"},
                                  {"mode": "PERMISSIVE", "resyncFraming": ""}])
def test_resync_framing_is_refused_before_any_file_is_read(opts):
    with pytest.raises(_native.IllegalArgumentException, match="resyncFraming"):
        tio._decoder_flags(opts, DATA)
    with pytest.raises(_native.IllegalArgumentException, match="resyncFraming"):
        tio.DefaultSource().buildReader(DATA, DATA, opts)
    with pytest.raises(_native.IllegalArgumentException, match="resyncFraming"):
        tio.DefaultSource().inferSchema(opts, ["/nonexistent/file.tfrecord"])


def test_header_bindings_and_jni_shim():
    hdr_ = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    m = re.search(r"#define\s+TFR_F_RESYNC\s+(0x[0-9a-fA-F]+)u", hdr_)
    assert m and int(m.group(1), 16) == A.TFR_F_RESYNC == 0x8
    assert re.search(r"int32_t\s+tfr_batch_dropped_spans\(tfr_batch\*,\s*int64_t\* n_dropped,\s*int64_t\* record,\s*int64_t\* offset,\s*"
                     r"int64_t\* nbytes,\s*int32_t\* code,\s*int32_t\* field,\s*int64_t cap\);", hdr_)
    assert "[11] lost regions and [12] the bytes in them" in hdr_
    L = _native.lib()
    assert "tfr_batch_dropped_spans" in _native.EXPORTS and hasattr(L, "tfr_batch_dropped_spans")
    assert L.tfr_batch_dropped_spans(None, None, None, None, None, None, None, 0) == A.TFR_E_INVALID_ARG
    src = os.path.join(ROOT, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    assert "Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchDroppedSpans" in open(src).read()
    p = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-DTFR_BUILD_JNI", "-I", os.path.join(ROOT, "tests", "jni_stub"),
                        "-I", os.path.join(ROOT, "include"), src], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
