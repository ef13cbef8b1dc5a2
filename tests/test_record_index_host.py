"""CPU tests of the record index (include/tfrgpu.h, RECORD INDEX; the DataSource option recordIndex=true): the option and its
refusals, parsing an index and detecting a stale one, isSplitable in every case, the C ABI's declarations and the JNI
mapping, and the checkpoint rule restated by tests/record_index.py against hand-made cases.  The GPU build, the seek and
the split reads: test_gpu_record_index.py."""
import os
import re
import struct

import pytest

import record_index as RX
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import LongType, StructField, StructType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCHEMA = StructType([StructField("x", LongType(), True)])


def frame_of(n):
    """one frame whose payload is n bytes (16 + n bytes in all)"""
    return pyref.frame(bytes(range(256)) * (n // 256) + bytes(n % 256))


# ---------------------------------------------------------------------------------------------
# the C ABI
# ---------------------------------------------------------------------------------------------
def test_declarations_and_status():
    hdr = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    assert re.search(r"TFR_E_INDEX_MISMATCH\s+= -19\b", hdr) and A.TFR_E_INDEX_MISMATCH == -19
    assert '#define TFR_INDEX_MAGIC            "TFRIDX01"' in hdr
    for s in ("tfr_indexer_create", "tfr_index_update", "tfr_index_result", "tfr_index_seek", "tfr_indexer_destroy"):
        assert s in _native.EXPORTS and hasattr(_native.lib(), s)
    assert _native.lib().tfr_status_string(A.TFR_E_INDEX_MISMATCH) == b"record index does not describe its file"
    assert isinstance(_native.error_for(A.TFR_E_INDEX_MISMATCH), _native.IOException)


def test_jni_maps_index_mismatch_to_ioexception():
    src = open(os.path.join(ROOT, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")).read()
    line = next(ln for ln in src.splitlines() if "TFR_E_INDEX_MISMATCH" in ln and "cls =" in ln)
    assert '"java/io/IOException"' in line
    for name in ("indexerCreate", "indexUpdate", "indexResult", "indexSeek", "indexerDestroy"):
        assert f"TfrGpu_{name}(" in src
    table = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert re.search(r"\|[^\n]*`TFR_E_INDEX_MISMATCH`[^\n]*`java\.io\.IOException`", table)


@pytest.mark.parametrize("stride", [0, 8, 15, 24, 1000, 1 << 31])
def test_bad_stride_is_refused_before_any_device_work(stride):
    with pytest.raises(_native.TfrError) as e:
        _native.Indexer(stride)
    assert e.value.code == A.TFR_E_INVALID_ARG


# ---------------------------------------------------------------------------------------------
# the option
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("v,want", [(None, False), ("false", False), ("FALSE", False), ("true", True), ("True", True), ("TRUE", True)])
def test_option_values(v, want):
    assert tio._record_index({} if v is None else {"recordIndex": v}) is want


@pytest.mark.parametrize("v", ["yes", "1", "", "on", " true"])
def test_bad_values_are_refused_before_any_work(v):
    for call in (lambda: tio.DefaultSource().prepareWrite({"recordIndex": v}, SCHEMA),
                 lambda: tio.DefaultSource().buildReader(SCHEMA, SCHEMA, {"recordIndex": v})):
        with pytest.raises(_native.IllegalArgumentException, match="recordIndex"):
            call()


@pytest.mark.parametrize("codec", ["gzip", "deflate", "bzip2", "org.apache.hadoop.io.compress.GzipCodec"])
def test_record_index_with_a_codec_is_refused(codec):
    with pytest.raises(_native.IllegalArgumentException, match="cannot be split"):
        tio.DefaultSource().prepareWrite({"recordIndex": "true", "codec": codec}, SCHEMA)
    tio.DefaultSource().prepareWrite({"recordIndex": "false", "codec": codec}, SCHEMA)     # the default stays as it was


def test_index_path():
    assert tio.index_path("/d/part-00000.tfrecord") == "/d/_part-00000.tfrecord.tfrindex"
    assert tio.index_path("x") == "_x.tfrindex"


# ---------------------------------------------------------------------------------------------
# the index file
# ---------------------------------------------------------------------------------------------
def test_parse_round_trip():
    data = b"".join(frame_of(n) for n in (5, 40, 0, 100))
    raw = RX.index_bytes(data, 32)
    n, stride, ck = tio.parse_index(raw, len(data))
    offs = RX.frames(data)
    assert (n, stride) == (4, 32)
    assert [tuple(map(int, c)) for c in ck] == RX.checkpoints(offs, len(data), 32)


@pytest.mark.parametrize("damage,match", [
    (lambda raw, size: (b"TFRIDX02" + raw[8:], size), "magic"),
    (lambda raw, size: (raw, size + 1), "describes"),
    (lambda raw, size: (raw, size - 1), "describes"),
    (lambda raw, size: (raw[:-16], size), "checkpoints"),
    (lambda raw, size: (raw + bytes(16), size), "checkpoints"),
    (lambda raw, size: (raw[:31], size), "header"),
    (lambda raw, size: (raw[:24] + struct.pack("<Q", 48) + raw[32:], size), "stride"),
    (lambda raw, size: (raw[:24] + struct.pack("<Q", 8) + raw[32:], size), "stride"),
])
def test_stale_or_damaged_index_is_refused(damage, match):
    data = b"".join(frame_of(n) for n in (5, 40, 0, 100))
    raw, size = damage(RX.index_bytes(data, 32), len(data))
    with pytest.raises(_native.IOException, match=match) as e:
        tio.parse_index(raw, size)
    assert e.value.code == A.TFR_E_INDEX_MISMATCH


# ---------------------------------------------------------------------------------------------
# isSplitable
# ---------------------------------------------------------------------------------------------
@pytest.fixture
def indexed(tmp_path):
    data = b"".join(frame_of(n) for n in range(0, 300, 7))
    p = tmp_path / "part-00000.tfrecord"
    p.write_bytes(data)
    open(tio.index_path(str(p)), "wb").write(RX.index_bytes(data, 64))
    return str(p), data


def test_is_splitable_only_with_everything_in_place(indexed, tmp_path):
    p, data = indexed
    ds = tio.DefaultSource()
    on = {"recordIndex": "true"}
    assert ds.isSplitable() is False
    assert ds.isSplitable(on, p) is True
    assert ds.isSplitable({"recordIndex": "TRUE", "mode": "DROPMALFORMED", "resyncFraming": "false"}, p) is True
    assert ds.isSplitable({}, p) is False
    assert ds.isSplitable({"recordIndex": "false"}, p) is False
    assert ds.isSplitable({"recordIndex": "maybe"}, p) is False
    assert ds.isSplitable({**on, "mode": "DROPMALFORMED", "resyncFraming": "true"}, p) is False
    assert ds.isSplitable({**on, "mode": "PERMISSIVE", "resyncFraming": "TRUE"}, p) is False
    # a compressed file, even with an index next to it
    gz = str(tmp_path / "part-00001.tfrecord.gz")
    open(gz, "wb").write(data)
    open(tio.index_path(gz), "wb").write(RX.index_bytes(data, 64))
    assert ds.isSplitable(on, gz) is False
    # no index, a bad magic, another size
    bare = str(tmp_path / "part-00002.tfrecord")
    open(bare, "wb").write(data)
    assert ds.isSplitable(on, bare) is False
    raw = RX.index_bytes(data, 64)
    open(tio.index_path(bare), "wb").write(b"TFRIDX00" + raw[8:])
    assert ds.isSplitable(on, bare) is False
    open(tio.index_path(bare), "wb").write(raw[:20])
    assert ds.isSplitable(on, bare) is False
    open(bare, "ab").write(b"\0")
    open(tio.index_path(bare), "wb").write(raw)
    assert ds.isSplitable(on, bare) is False


# ---------------------------------------------------------------------------------------------
# the checkpoint rule, hand-made cases
# ---------------------------------------------------------------------------------------------
def test_empty_file():
    assert RX.frames(b"") == [] and RX.checkpoints([], 0, 16) == []
    assert RX.index_bytes(b"", 16) == b"TFRIDX01" + struct.pack("<QQQ", 0, 0, 16)
    assert RX.seek([], 0, 0) == (0, 0)


def test_one_record():
    data = frame_of(20)                          # 36 bytes: slots 0, 1, 2 at stride 16
    assert RX.checkpoints(RX.frames(data), 36, 16) == [(0, 0), (36, 1), (36, 1)]
    assert RX.checkpoints(RX.frames(data), 36, 64) == [(0, 0)]


def test_record_larger_than_the_stride():
    data = frame_of(10) + frame_of(100) + frame_of(0)      # frames at 0, 26, 142; 158 bytes
    assert RX.frames(data) == [0, 26, 142]
    assert RX.checkpoints([0, 26, 142], 158, 16) == [(0, 0), (26, 1), (142, 2), (142, 2), (142, 2), (142, 2), (142, 2),
                                                     (142, 2), (142, 2), (158, 3)]


def test_records_ending_on_stride_boundaries():
    data = frame_of(16) + frame_of(0) + frame_of(16)       # frames at 0, 32, 48; 80 bytes
    assert RX.checkpoints(RX.frames(data), 80, 16) == [(0, 0), (32, 1), (32, 1), (48, 2), (80, 3)]
    assert RX.checkpoints(RX.frames(data), 80, 32) == [(0, 0), (32, 1), (80, 3)]


def test_last_checkpoint_past_the_last_frame():
    data = frame_of(0) + frame_of(100)                     # frames at 0, 16; 132 bytes
    ck = RX.checkpoints(RX.frames(data), 132, 16)
    assert len(ck) == 9 and ck[0] == (0, 0) and ck[1] == (16, 1) and ck[2:] == [(132, 2)] * 7
    assert RX.checkpoints(RX.frames(data), 132, 128) == [(0, 0), (132, 2)]
    # stray bytes after the last frame (a clean end of file) count in data_bytes
    assert RX.checkpoints(RX.frames(data + b"\0" * 5), 137, 16)[-1] == (137, 2)


def test_seek_and_split_rule():
    offs, size = [0, 26, 142], 158
    assert [RX.seek(offs, size, t) for t in (0, 1, 26, 27, 142, 143, 158)] == [(0, 0), (1, 26), (1, 26), (2, 142), (2, 142), (3, 158), (3, 158)]
    # every frame is in exactly one split, wherever the cuts are
    for cuts in ([0, 158], [0, 1, 158], [0, 26, 27, 142, 158], list(range(159))):
        got = [i for s, e in zip(cuts, cuts[1:]) for i in RX.split(offs, s, e)]
        assert got == [0, 1, 2]


def test_framing_error_gives_no_index():
    data = frame_of(10) + frame_of(10)
    bad = bytearray(data)
    bad[26 + 9] ^= 1                              # the second frame's length CRC
    with pytest.raises(RX.FramingError) as e:
        RX.index_bytes(bytes(bad), 16)
    assert (e.value.code, e.value.offset) == (A.TFR_E_CRC_LENGTH, 26)
