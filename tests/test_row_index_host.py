"""CPU tests of the generated fields TFR_T_ROW_INDEX and TFR_T_RECORD_OFFSET (include/tfrgpu.h, POSITIONS; Spark's
`_metadata.row_index`): schema validation and lowering, the encoder's refusal, the argument errors of the `_at` calls and of
tfr_batch_extent, io.py's mapping of Spark's temporary metadata columns, the JNI shim, and the entry rule restated by
tests/position_walk.py, pinned clause by clause and over random block cuts.  The decode itself: test_gpu_row_index.py."""
import os
import random
import re
import struct
import subprocess

import pytest

import position_walk as PW
import resync_walk as RW
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import (ArrayType, BinaryType, LongType, RecordOffsetType, RowIndexType, StringType,
                                          StructField, StructType)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C = _native.C


def fields(*fs):
    return StructType([StructField(*f) for f in fs])


def create(sch, rt=0):
    """-> (status, number of fields or the error text)"""
    try:
        s = _native.Schema(sch, rt)
    except _native.TfrError as e:
        return e.code, str(e)
    try:
        return 0, _native.lib().tfr_schema_num_fields(s.h)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------
# the C ABI: constants, schema validation, the encoder, argument errors
# ---------------------------------------------------------------------------------------------
def test_constants_and_symbols_in_the_header():
    hdr = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    assert re.search(r"TFR_T_ROW_INDEX\s+= 8\b", hdr) and re.search(r"TFR_T_RECORD_OFFSET = 9\b", hdr)
    assert A.TFR_T_ROW_INDEX == 8 and A.TFR_T_RECORD_OFFSET == 9
    assert re.search(r"int32_t tfr_decode_at\(tfr_decoder\*, const void\* data, size_t nbytes, int32_t data_on_device, int32_t is_final,\s*"
                     r"int64_t first_entry, int64_t first_offset, tfr_batch\*\* out, size_t\* consumed\);", hdr)
    assert re.search(r"int32_t tfr_decode_submit_at\(tfr_decoder\*, const void\* data, size_t nbytes, int32_t data_on_device, int32_t is_final,\s*"
                     r"int64_t first_entry, int64_t first_offset, tfr_batch\*\* out\);", hdr)
    assert "int32_t tfr_batch_extent(tfr_batch*, size_t* consumed, int64_t* entries);" in hdr
    for s in ("tfr_decode_at", "tfr_decode_submit_at", "tfr_batch_extent"):
        assert s in _native.EXPORTS and hasattr(_native.lib(), s)


@pytest.mark.parametrize("t", [RowIndexType(), RecordOffsetType()])
@pytest.mark.parametrize("pos", [0, 1, 2])
def test_generated_field_anywhere_at_depth_0(t, pos):
    fs = [StructField("a", LongType()), StructField("s", StringType())]
    fs.insert(pos, StructField("gen", t, False))
    assert create(StructType(fs)) == (0, 3)
    assert create(fields(("ri", RowIndexType()), ("ro", RecordOffsetType()))) == (0, 2)


@pytest.mark.parametrize("t", [RowIndexType(), RecordOffsetType()])
@pytest.mark.parametrize("depth", [1, 2])
def test_generated_field_below_depth_0_is_refused(t, depth):
    dt = t
    for _ in range(depth):
        dt = ArrayType(dt)
    code, msg = create(fields(("a", LongType()), ("gen", dt)), 1)
    assert code == A.TFR_E_UNSUPPORTED_TYPE and "'gen'" in msg and "depth 0" in msg


@pytest.mark.parametrize("t", [RowIndexType(), RecordOffsetType()])
def test_two_of_one_kind_are_refused(t):
    code, msg = create(fields(("g1", t), ("a", LongType()), ("g2", t)))
    assert code == A.TFR_E_UNSUPPORTED_TYPE and "'g2'" in msg and "at most one" in msg
    code, msg = create(fields(("g1", t), ("g2", t)), 2)                   # ByteArray too
    assert code == A.TFR_E_UNSUPPORTED_TYPE and "'g2'" in msg


def test_a_generated_field_takes_part_in_the_duplicate_name_check():
    code, msg = create(fields(("x", RowIndexType()), ("x", LongType())))
    assert code == A.TFR_E_INVALID_ARG and "duplicate" in msg


def test_byte_array_appends_the_generated_fields():
    """byteArray first, then the generated fields in the caller's order; every other field stays ignored"""
    assert create(fields(("x", StringType()), ("y", ArrayType(LongType()))), 2) == (0, 1)
    assert create(fields(("x", StringType()), ("ro", RecordOffsetType()), ("y", LongType()), ("ri", RowIndexType())), 2) == (0, 3)
    assert create(fields(("ri", RowIndexType())), 2) == (0, 2)


def test_encoder_refuses_a_generated_field():
    """before any device work: a writer never gets a metadata column"""
    for rt, sch in [(0, fields(("a", LongType()), ("ri", RowIndexType()))), (1, fields(("ro", RecordOffsetType()))),
                    (2, fields(("ri", RowIndexType())))]:
        s = _native.Schema(sch, rt)
        out = C.c_void_p()
        assert _native.lib().tfr_encoder_create(s.h, 0, 0, C.byref(out)) == A.TFR_E_UNSUPPORTED_TYPE and not out.value
        assert "cannot be written" in _native.lib().tfr_last_error().decode()
        s.close()


def test_at_calls_and_extent_refuse_null_handles():
    L = _native.lib()
    b, used, n = C.c_void_p(), C.c_size_t(), C.c_int64()
    assert L.tfr_decode_at(None, None, 0, 0, 1, 0, 0, C.byref(b), C.byref(used)) == A.TFR_E_INVALID_ARG
    assert L.tfr_decode_submit_at(None, None, 0, 0, 1, 0, 0, C.byref(b)) == A.TFR_E_INVALID_ARG
    assert L.tfr_decode_submit_at(None, None, 0, 0, 1, -1, -1, C.byref(b)) == A.TFR_E_INVALID_ARG
    assert L.tfr_batch_extent(None, C.byref(used), C.byref(n)) == A.TFR_E_INVALID_ARG
    assert L.tfr_batch_extent(None, None, None) == A.TFR_E_INVALID_ARG
    assert not b.value


# ---------------------------------------------------------------------------------------------
# io.py and the JNI shim
# ---------------------------------------------------------------------------------------------
def test_read_file_maps_the_temporary_metadata_columns():
    req = fields(("a", LongType()), ("_tmp_metadata_row_index", LongType(), False), ("s", StringType()),
                 ("_tmp_metadata_record_offset", LongType(), False))
    got = tio._decoder_schema(req)
    assert [f.name for f in got] == req.names
    assert [type(f.dataType) for f in got] == [LongType, RowIndexType, StringType, RecordOffsetType]
    # another type under the name is a data field, and so is any other name
    other = fields(("_tmp_metadata_row_index", StringType()), ("row_index", LongType()))
    assert [f.dataType for f in tio._decoder_schema(other)] == [StringType(), LongType()]


def test_metadata_schema_fields():
    got = tio.DefaultSource().metadataSchemaFields()
    assert got == [("row_index", "_tmp_metadata_row_index", LongType()), ("record_offset", "_tmp_metadata_record_offset", LongType())]
    assert tio.DefaultSource().isSplitable() is False


def test_jni_shim_binds_the_position_calls():
    src = os.path.join(ROOT, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    text = open(src).read()
    for name, call in [("decodeAt", "tfr_decode_at("), ("decodeSubmitAt", "tfr_decode_submit_at("), ("batchExtent", "tfr_batch_extent(")]:
        assert "Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_" + name + "(" in text and call in text
    p = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-DTFR_BUILD_JNI", "-I", os.path.join(ROOT, "tests", "jni_stub"),
                        "-I", os.path.join(ROOT, "include"), src], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr


# ---------------------------------------------------------------------------------------------
# the entry rule (position_walk), clause by clause and over random block cuts
# ---------------------------------------------------------------------------------------------
def frame(payload, good=True):
    f = pyref.frame(payload)
    return f if good else f[:-4] + struct.pack("<I", struct.unpack("<I", f[-4:])[0] ^ 1)


def payload_crc_fails(payload, crc):
    return pyref.masked_crc32c(payload) != struct.unpack("<I", crc)[0]


def corpus(seed, n=60, n_bad=6, n_damaged=3):
    """frames of random sizes, n_bad of them with a failing payload CRC, n_damaged with a flipped length-CRC bit"""
    R = random.Random(seed)
    frames = [frame(R.randbytes(R.randrange(0, 90))) for _ in range(n)]
    bad = set(R.sample(range(n), n_bad))
    for i in bad:
        frames[i] = frame(frames[i][12:-4], False)
    damaged = R.sample(range(1, n), n_damaged)
    for i in damaged:
        f = bytearray(frames[i])
        f[8 + R.randrange(4)] ^= 1 << R.randrange(8)
        frames[i] = bytes(f)
    return b"".join(frames), frames, bad, set(damaged)


def offsets(frames):
    out, o = [], 0
    for f in frames:
        out.append(o)
        o += len(f)
    return out


def test_failfast_without_errors_is_first_entry_plus_r():
    data, frames, _, _ = corpus(1, n_bad=0, n_damaged=0)
    got, (used, n) = PW.block(data, True, False, PW.FAILFAST, payload_crc_fails, 1000, 77)
    assert got == [(1000 + r, 77 + o) for r, o in enumerate(offsets(frames))]
    assert (used, n) == (len(data), len(frames))


def test_failfast_stops_in_front_of_the_first_failing_record():
    data, frames, bad, _ = corpus(2, n_damaged=0)
    got, (used, n) = PW.block(data, True, False, PW.FAILFAST, payload_crc_fails)
    k = min(bad)
    assert got == list(zip(range(k), offsets(frames)[:k])) and (used, n) == (offsets(frames)[k], k)


def test_dropmalformed_skips_exactly_the_dropped_entries():
    data, frames, bad, _ = corpus(3, n_damaged=0)
    got, (used, n) = PW.block(data, True, False, PW.DROPMALFORMED, payload_crc_fails, 5, 0)
    idx = [r for r, _ in got]
    assert all(a < b for a, b in zip(idx, idx[1:]))
    assert set(range(5, 5 + len(frames))) - set(idx) == {5 + i for i in bad}
    assert [o for _, o in got] == [offsets(frames)[i - 5] for i in idx]
    assert (used, n) == (len(data), len(frames))                      # dropped frames count as entries


def test_permissive_corrupt_rows_are_their_dropped_record_plus_the_base():
    data, frames, bad, _ = corpus(4)
    ents, _ = PW.entries(data, True, True)
    got, _ = PW.block(data, True, True, PW.PERMISSIVE, payload_crc_fails, 10, 1 << 33)
    assert len(got) == len(ents)                                        # every entry is a row
    dropped = sorted(PW.frame_bad(data, payload_crc_fails)(ents))       # what tfr_batch_dropped lists: (record, offset)
    assert dropped and any(ents[k][0] == "region" for k in dropped)
    for k in dropped:
        assert got[k] == (10 + k, (1 << 33) + ents[k][1])


def test_a_lost_region_is_one_entry_at_its_first_byte():
    data, frames, bad, damaged = corpus(5, n_bad=0)
    ents, _ = PW.entries(data, True, True)
    regions = [e for e in ents if e[0] == "region"]
    assert regions and all(e[1] in offsets(frames) for e in regions)   # a region starts at the header whose length CRC failed
    got, _ = PW.block(data, True, True, PW.DROPMALFORMED, payload_crc_fails)
    kept = {o for _, o in got}
    assert all(e[1] not in kept for e in regions)
    assert [r for r, _ in got] == [k for k, e in enumerate(ents) if e[0] == "frame"]


def test_without_resync_a_framing_stop_ends_the_entries():
    data, frames, bad, damaged = corpus(6, n_bad=0, n_damaged=1)
    ents, consumed = PW.entries(data, True, False)
    k = min(damaged)
    assert len(ents) == k and consumed == offsets(frames)[k]


@pytest.mark.parametrize("mode, resync", [(PW.FAILFAST, False), (PW.DROPMALFORMED, False), (PW.PERMISSIVE, False),
                                          (PW.DROPMALFORMED, True), (PW.PERMISSIVE, True)])
@pytest.mark.parametrize("seed", range(8))
def test_values_do_not_depend_on_where_blocks_are_cut(mode, resync, seed):
    data, frames, bad, damaged = corpus(100 + seed, n_damaged=3 if resync else 0)
    whole, _ = PW.block(data, True, resync, mode, payload_crc_fails)
    R = random.Random(seed)
    for _ in range(6):
        cuts = sorted(R.sample(range(1, len(data)), R.randrange(1, 12)))
        assert PW.stream(data, cuts, resync, mode, payload_crc_fails) == whole, cuts


def test_the_walk_is_resync_walks_walk():
    data, *_ = corpus(7)
    assert PW.entries(data, True, True) == RW.walk(data, True)
    assert PW.entries(data[:-3], False, True) == RW.walk(data[:-3], False)


# ---------------------------------------------------------------------------------------------
# the C emulator of the block loop with positions (tests/emulator/position_emulator.c)
# ---------------------------------------------------------------------------------------------
EMULATOR = os.path.join(ROOT, "tests", "emulator", "position_emulator.c")


def build_position_emulator(exe):
    import __graft_entry__ as g
    g.build()
    pkg = os.path.join(ROOT, "spark-tfrecord_b200")
    cmd = ["gcc", "-std=c11", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), EMULATOR, "-o", exe,
           "-L", pkg, "-l:libtfrgpu.so", f"-Wl,-rpath,{pkg}"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr[-3000:]
    return exe


def test_position_emulator_builds_against_the_header_alone_and_runs_its_device_free_checks(tmp_path):
    exe = build_position_emulator(str(tmp_path / "positions"))
    includes = [l.strip() for l in open(EMULATOR).read().splitlines() if l.strip().startswith("#include")]
    assert all(i.startswith("#include <std") or i in ('#include "tfrgpu.h"', "#include <string.h>") for i in includes), includes
    p = subprocess.run([exe, "abi"], capture_output=True, text=True, timeout=60)
    assert p.returncode == 0, p.stderr
    out = p.stdout.splitlines()
    assert out[0] == "abi 2" and out[-1] == "staging slots 3"
    p = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert p.returncode == 2 and "positions FILE BLOCK MODE" in p.stderr
