"""CPU tests of drop mode's host side: the `mode` option of the reader (Spark's ParseMode names, case-insensitive), the
flag and the new C symbol in the header, the bindings and the JNI shim.  The decode itself: test_gpu_drop_malformed.py."""
import os
import re

import pytest

from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import LongType, StructField, StructType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("options, flags", [
    (None, A.TFR_F_DEFAULT), ({}, A.TFR_F_DEFAULT), ({"mode": "FAILFAST"}, A.TFR_F_DEFAULT), ({"mode": "failFast"}, A.TFR_F_DEFAULT),
    ({"mode": "DROPMALFORMED"}, A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED),
    ({"mode": "dropmalformed"}, A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED),
    ({"mode": "DropMalformed", "recordType": "SequenceExample"}, A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED),
])
def test_mode_option(options, flags):
    assert tio._decoder_flags(options) == flags


def test_permissive_is_refused():
    for mode in ("PERMISSIVE", "permissive"):
        with pytest.raises(_native.IllegalArgumentException, match="corrupt-record column"):
            tio._decoder_flags({"mode": mode})


@pytest.mark.parametrize("mode", ["", "DROP", "FAIL_FAST", "ignore"])
def test_unknown_mode_is_refused(mode):
    with pytest.raises(_native.IllegalArgumentException, match="FAILFAST and DROPMALFORMED"):
        tio._decoder_flags({"mode": mode})


def test_reader_checks_the_mode_before_reading():
    """buildReader (and with it DefaultSource.load) refuses a bad mode before it opens a file or a device"""
    sch = StructType([StructField("a", LongType())])
    with pytest.raises(_native.IllegalArgumentException):
        tio.DefaultSource().buildReader(sch, sch, {"mode": "PERMISSIVE"})
    with pytest.raises(_native.IllegalArgumentException):
        tio.DefaultSource().load(os.path.join(ROOT, "tests", "golden", "frame_ok.tfrecord"), sch, {"mode": "bogus"})


def test_flag_and_symbol_in_the_header():
    hdr = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    m = re.search(r"#define\s+TFR_F_DROP_MALFORMED\s+(0x[0-9a-fA-F]+)u", hdr)
    assert m and int(m.group(1), 16) == A.TFR_F_DROP_MALFORMED == 0x2
    assert A.TFR_F_DEFAULT & A.TFR_F_DROP_MALFORMED == 0            # FAILFAST stays the default
    assert re.search(r"int32_t\s+tfr_batch_dropped\(tfr_batch\*,\s*int64_t\* n_dropped,", hdr)
    assert "tfr_batch_dropped" in _native.EXPORTS
    assert "[9] records dropped" in hdr
    assert set(A.RECORD_ERRORS) == {A.TFR_E_CRC_DATA, A.TFR_E_MALFORMED_PROTO, A.TFR_E_KIND_MISMATCH, A.TFR_E_EMPTY_SCALAR,
                                    A.TFR_E_NULL_IN_NONNULL, A.TFR_E_BAD_NESTING}


def test_library_exports_the_symbol():
    L = _native.lib()
    assert hasattr(L, "tfr_batch_dropped")
    assert L.tfr_batch_dropped(None, None, None, None, None, None, 0) == A.TFR_E_INVALID_ARG


def test_jni_shim_has_batch_dropped():
    src = open(os.path.join(ROOT, "spark-tfrecord_b200", "jni", "tfrgpu_jni.cpp")).read()
    assert "Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_batchDropped" in src
    assert "tfr_batch_dropped(" in src
