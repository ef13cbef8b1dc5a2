"""CPU tests of PERMISSIVE's host side: the `mode` option with and without a corrupt-record column in the data schema
(Spark's columnNameOfCorruptRecord, default _corrupt_record), its type checks, ByteArray records, the flag and the new C
symbol in the header, the argument errors of tfr_decoder_create_permissive, the bindings and the JNI shim.  The decode
itself: test_gpu_permissive.py."""
import os
import re
import subprocess

import pytest

from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import (ArrayType, BinaryType, LongType, StringType, StructField, StructType)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERMISSIVE = A.TFR_F_DEFAULT | A.TFR_F_PERMISSIVE


def schema(*fields):
    return StructType([StructField(*f) for f in fields])


DATA = schema(("a", LongType()), ("_corrupt_record", BinaryType()), ("s", StringType()))


@pytest.mark.parametrize("mode", ["PERMISSIVE", "permissive", "Permissive"])
def test_mode_with_a_corrupt_column(mode):
    assert tio._decoder_flags({"mode": mode}, DATA) == PERMISSIVE
    assert tio._read_mode({"mode": mode}, DATA, DATA) == (PERMISSIVE, 1)
    assert A.TFR_F_PERMISSIVE & (A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED) == 0


def test_mode_with_a_named_corrupt_column():
    sch = schema(("bad", BinaryType()), ("a", LongType()))
    opts = {"mode": "PERMISSIVE", "columnNameOfCorruptRecord": "bad"}
    assert tio._read_mode(opts, sch, sch) == (PERMISSIVE, 0)
    with pytest.raises(_native.IllegalArgumentException, match="corrupt-record column"):
        tio._decoder_flags({"mode": "PERMISSIVE"}, sch)                 # the default name is not in the schema


def test_pruned_corrupt_column():
    """the projection dropped the column: failing records still become rows (of nulls), and no field is passed"""
    required = schema(("s", StringType()), ("a", LongType()))
    assert tio._read_mode({"mode": "PERMISSIVE"}, DATA, required) == (PERMISSIVE, None)
    assert tio._read_mode({"mode": "PERMISSIVE"}, DATA, schema(("_corrupt_record", BinaryType()))) == (PERMISSIVE, 0)


def test_other_modes_pass_no_corrupt_column():
    assert tio._read_mode({}, DATA, DATA) == (A.TFR_F_DEFAULT, None)
    assert tio._read_mode({"mode": "DROPMALFORMED"}, DATA, DATA) == (A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED, None)


@pytest.mark.parametrize("sch", [schema(("a", LongType())), None, StructType()])
def test_permissive_without_a_corrupt_column_is_refused(sch):
    with pytest.raises(_native.IllegalArgumentException, match="corrupt-record column"):
        tio._decoder_flags({"mode": "PERMISSIVE"}, sch)
    with pytest.raises(_native.IllegalArgumentException, match="corrupt-record column"):
        tio.DefaultSource().buildReader(sch or StructType(), sch or StructType(), {"mode": "PERMISSIVE"})


@pytest.mark.parametrize("field", [StructField("_corrupt_record", StringType()), StructField("_corrupt_record", LongType()),
                                   StructField("_corrupt_record", ArrayType(BinaryType())),
                                   StructField("_corrupt_record", BinaryType(), False)])
def test_wrong_corrupt_column_is_refused(field):
    sch = StructType([StructField("a", LongType()), field])
    with pytest.raises(_native.IllegalArgumentException, match="_corrupt_record"):
        tio._decoder_flags({"mode": "PERMISSIVE"}, sch)
    with pytest.raises(_native.IllegalArgumentException, match="binary type and nullable"):
        tio.DefaultSource().buildReader(sch, sch, {"mode": "PERMISSIVE"})


def test_byte_array_is_refused():
    with pytest.raises(_native.IllegalArgumentException, match="ByteArray"):
        tio._decoder_flags({"mode": "PERMISSIVE", "recordType": "ByteArray"}, DATA)
    assert tio._decoder_flags({"mode": "PERMISSIVE", "recordType": "SequenceExample"}, DATA) == PERMISSIVE


def test_read_file_checks_the_mode_before_reading():
    """readFile called directly takes its schema as the data schema: without the column it refuses before it opens the file or a device"""
    sch = schema(("a", LongType()))
    ok = tio.PartitionedFile(os.path.join(ROOT, "tests", "golden", "frame_ok.tfrecord"))
    with pytest.raises(_native.IllegalArgumentException, match="corrupt-record column"):
        tio.TFRecordFileReader.readFile(None, {"mode": "PERMISSIVE"}, ok, sch)


def test_flag_and_symbol_in_the_header():
    hdr = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    m = re.search(r"#define\s+TFR_F_PERMISSIVE\s+(0x[0-9a-fA-F]+)u", hdr)
    assert m and int(m.group(1), 16) == A.TFR_F_PERMISSIVE == 0x4
    assert re.search(r"int32_t\s+tfr_decoder_create_permissive\(const tfr_schema\*,\s*int32_t device,\s*uint32_t flags,\s*"
                     r"int32_t corrupt_field,\s*tfr_decoder\*\* out\);", hdr)
    assert "tfr_decoder_create_permissive" in _native.EXPORTS
    assert "[10] records delivered as corrupt rows" in hdr and "n <= 11 gets them all, counter [10] being" in hdr
    assert re.search(r"#define\s+TFR_ABI_VERSION\s+2\b", hdr)


def test_create_permissive_argument_errors():
    """argument errors come back before any device work (no GPU is needed to see them)"""
    L = _native.lib()
    out = _native.C.c_void_p()
    assert L.tfr_decoder_create_permissive(None, 0, PERMISSIVE, -1, _native.C.byref(out)) == A.TFR_E_INVALID_ARG
    assert L.tfr_decoder_create_permissive(None, 0, PERMISSIVE, 0, None) == A.TFR_E_INVALID_ARG
    assert L.tfr_decoder_create_permissive(None, 0, A.TFR_F_DEFAULT, -1, _native.C.byref(out)) == A.TFR_E_INVALID_ARG
    assert not out.value


def _schema_handle(sch, rt=0):
    return _native.Schema(sch, rt)


@pytest.mark.parametrize("flags, field, what", [
    (PERMISSIVE | A.TFR_F_DROP_MALFORMED, -1, "exclude each other"),
    (PERMISSIVE | A.TFR_F_DROP_MALFORMED, 1, "exclude each other"),
    (A.TFR_F_DEFAULT, 1, "TFR_F_PERMISSIVE"),
    (PERMISSIVE, 0, "'a'"),                     # LongType
    (PERMISSIVE, 2, "'s'"),                     # StringType
    (PERMISSIVE, 3, "'nn'"),                    # not nullable
    (PERMISSIVE, 4, "'arr'"),                   # array of binary
    (PERMISSIVE, 5, "no such schema field"),
    (PERMISSIVE, -2, "no such schema field"),
])
def test_create_permissive_refuses_before_device_work(flags, field, what):
    sch = schema(("a", LongType()), ("_corrupt_record", BinaryType()), ("s", StringType()), ("nn", BinaryType(), False),
                 ("arr", ArrayType(BinaryType())))
    S = _schema_handle(sch)
    out = _native.C.c_void_p()
    rc = _native.lib().tfr_decoder_create_permissive(S.h, 0, flags, field, _native.C.byref(out))
    assert rc == A.TFR_E_INVALID_ARG and not out.value
    assert what in _native.lib().tfr_last_error().decode()


def test_create_refuses_both_modes_and_byte_array():
    out = _native.C.c_void_p()
    S = _schema_handle(DATA)
    assert _native.lib().tfr_decoder_create(S.h, 0, PERMISSIVE | A.TFR_F_DROP_MALFORMED, _native.C.byref(out)) == A.TFR_E_INVALID_ARG
    B = _schema_handle(StructType(), 2)
    assert _native.lib().tfr_decoder_create(B.h, 0, PERMISSIVE, _native.C.byref(out)) == A.TFR_E_INVALID_ARG
    assert "ByteArray" in _native.lib().tfr_last_error().decode()
    assert _native.lib().tfr_decoder_create_permissive(B.h, 0, PERMISSIVE, -1, _native.C.byref(out)) == A.TFR_E_INVALID_ARG
    assert not out.value


def test_stats_names_the_new_counter():
    src = open(os.path.join(ROOT, "spark-tfrecord_b200", "_native.py")).read()
    assert '"records_dropped", "records_corrupt"]' in src


def test_jni_shim_has_decoder_create_permissive():
    src = os.path.join(ROOT, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")
    text = open(src).read()
    assert "Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_decoderCreatePermissive" in text
    assert "tfr_decoder_create_permissive(" in text
    p = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-DTFR_BUILD_JNI", "-I", os.path.join(ROOT, "tests", "jni_stub"),
                        "-I", os.path.join(ROOT, "include"), src], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
