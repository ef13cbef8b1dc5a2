"""Checks of the pipelined encode's C ABI that need no GPU: the pipeline depth, argument errors of tfr_encode_rows_submit,
tfr_encoded_wait, tfr_encoded_result and tfr_encoder_get_stats for null handles or outputs, tfr_encoded_release(NULL), and the C
emulator of the pipelined RowWriter (tests/emulator/rowwrite_emulator.c, `rowwrite`) building against include/tfrgpu.h.  The helpers below also give the
emulator's schema and rows to the GPU test of `rowwrite` (test_gpu_encode_rows_pipelined.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "spark-tfrecord_b200")
SRC = os.path.join(ROOT, "tests", "emulator", "rowwrite_emulator.c")


def build_emulator(exe):
    import __graft_entry__ as g
    g.build()
    cmd = ["gcc", "-std=c11", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), SRC, "-o", exe,
           "-L", PKG, "-l:libtfrgpu.so", f"-Wl,-rpath,{PKG}"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr[-3000:]
    return exe


def emulator_schema():
    from spark_tfrecord_b200.sqltypes import ArrayType, FloatType, LongType, StringType, StructField, StructType
    return StructType([StructField("id", LongType(), nullable=False), StructField("w", FloatType()), StructField("name", StringType()),
                       StructField("emb", ArrayType(FloatType()))])


def emulator_rows(n):
    """the rows of the emulator's generator (row_value_* in rowwrite_emulator.c, the same as in fileformat_emulator.c)"""
    f = np.float32
    return [(i * i - 7 * i - 3, f(i) * f(0.5) - f(100.0), None if i % 11 == 5 else f"row-{i}-{'x' if i % 3 else 'yy'}",
             [f(i + k) * f(0.25) for k in range(i % 6)]) for i in range(n)]


@pytest.fixture(scope="module")
def L():
    from spark_tfrecord_b200 import _native
    return _native.lib()


def test_emulator_with_rowwrite_builds(tmp_path):
    exe = build_emulator(str(tmp_path / "emu"))
    p = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert p.returncode == 2 and "rowwrite DIR N_ROWS FLUSH_ROWS" in p.stderr


def test_num_row_slots_is_the_pipeline_depth(L):
    assert L.tfr_encoder_num_row_slots() == 3


def test_null_handles_and_outputs_are_invalid_arg(L):
    from spark_tfrecord_b200 import _cabi as A
    h = C.c_void_p()
    rows = np.zeros(8, np.uint8)
    offs = np.array([0, 8], np.int32)
    assert L.tfr_encode_rows_submit(None, rows.ctypes.data, offs.ctypes.data, 1, 0, C.byref(h)) == A.TFR_E_INVALID_ARG
    assert L.tfr_encode_rows_submit(None, rows.ctypes.data, offs.ctypes.data, 1, 0, None) == A.TFR_E_INVALID_ARG
    er = C.c_int64()
    assert L.tfr_encoded_wait(None, C.byref(er)) == A.TFR_E_INVALID_ARG
    p, nb = C.c_void_p(), C.c_size_t()
    assert L.tfr_encoded_result(None, 1, C.byref(p), C.byref(nb)) == A.TFR_E_INVALID_ARG
    assert L.tfr_encoded_result(None, 0, None, None) == A.TFR_E_INVALID_ARG
    v = (C.c_int64 * 8)()
    assert L.tfr_encoder_get_stats(None, v, 8) == A.TFR_E_INVALID_ARG
    assert L.tfr_encoder_get_stats(None, None, 8) == A.TFR_E_INVALID_ARG
    assert L.tfr_encoder_row_staging_slot(None, 0, 16, C.byref(p), None) == A.TFR_E_INVALID_ARG


def test_release_of_null_is_a_no_op(L):
    L.tfr_encoded_release(None)
