"""Checks of tfr_batch_rows_async that need no GPU: its argument errors (a null batch, bad partition rows, checked before the
batch), the symbol and its binding, the decoder counters' new bound, the C emulator of the row-reading BlockIterator
(tests/emulator/rowread_emulator.c) building against include/tfrgpu.h alone and passing its device-free checks, and the JNI
shim's new entry points.  The emulator's GPU run is in test_gpu_decode_rows_pipelined.py."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "spark-tfrecord_b200")
SRC = os.path.join(ROOT, "tests", "emulator", "rowread_emulator.c")


def build_rowread(exe):
    import __graft_entry__ as g
    g.build()
    cmd = ["gcc", "-std=c11", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), SRC, "-o", exe,
           "-L", PKG, "-l:libtfrgpu.so", f"-Wl,-rpath,{PKG}"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr[-3000:]
    return exe


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from spark_tfrecord_b200 import _native
    return _native.lib()


def _last_error(L):
    return (L.tfr_last_error() or b"").decode()


def test_symbol_is_exported_and_bound(L):
    from spark_tfrecord_b200 import _native
    out = subprocess.run(["nm", "-D", "--defined-only", _native.LIB_PATH], capture_output=True, text=True).stdout
    assert re.search(r" T tfr_batch_rows_async\b", out)
    assert "tfr_batch_rows_async" in _native.EXPORTS
    assert hasattr(_native.Batch, "unsafe_rows_async")


def test_null_batch_is_invalid_arg(L):
    from spark_tfrecord_b200 import _cabi as A
    assert L.tfr_batch_rows_async(None, 1, None, 0, 0, None) == A.TFR_E_INVALID_ARG
    assert "null batch" in _last_error(L)
    assert L.tfr_batch_rows_async(None, 0, None, 0, 0, None) == A.TFR_E_INVALID_ARG


@pytest.mark.parametrize("row,np_,flags,msg", [
    (bytes(8), 1, b"\0", "fixed region"),                                   # 1 field: 8 null bytes + 8 slot bytes at least
    (bytes(12), 0, None, "without fields"),                                  # bytes but no fields
    (bytes(16), 1, None, "null partition row or variable-slot flags"),       # flags missing
    (bytes(20), 1, b"\0", "not a multiple of 8"),
    ((2).to_bytes(8, "little") + bytes(8), 1, b"\0", "null bit set"),       # bit 1 set, one field
    (bytes(8) + ((8 << 32) | 8).to_bytes(8, "little"), 1, b"\1", "variable slot"),   # offset inside the fixed region
    (bytes(16), 5000, b"\0" * 5000, "outside 0..4096"),
])
def test_bad_partition_rows_are_invalid_arg_before_the_batch(L, row, np_, flags, msg):
    from spark_tfrecord_b200 import _cabi as A
    assert L.tfr_batch_rows_async(None, 1, row, len(row), np_, flags) == A.TFR_E_INVALID_ARG
    assert msg in _last_error(L), _last_error(L)


def test_stats_take_ten_counters(L):
    from spark_tfrecord_b200 import _cabi as A
    v = (C.c_int64 * 10)()
    assert L.tfr_decoder_get_stats(None, v, 10) == A.TFR_E_INVALID_ARG
    hdr = open(os.path.join(ROOT, "include", "tfrgpu.h")).read()
    assert "n /* <= 10 */" in hdr and "tfr_batch_rows_async(tfr_batch*" in hdr


def test_rowread_emulator_builds_and_runs_its_device_free_checks(tmp_path):
    exe = build_rowread(str(tmp_path / "rowread"))
    src = open(SRC).read()
    includes = [l.strip() for l in src.splitlines() if l.strip().startswith("#include")]
    assert '#include "tfrgpu.h"' in includes
    assert all(i.startswith("#include <std") or i in ('#include "tfrgpu.h"', "#include <string.h>") for i in includes), includes
    p = subprocess.run([exe, "abi"], capture_output=True, text=True, timeout=60)
    assert p.returncode == 0, p.stderr
    out = p.stdout.splitlines()
    assert out[0] == "abi 2" and out[-1] == "staging slots 3"
    p = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert p.returncode == 2 and "rowread FILE BLOCK" in p.stderr


def test_jni_shim_declares_the_async_rows_calls():
    src = os.path.join(PKG, "jni", "tfrgpu_jni.cpp")
    p = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-DTFR_BUILD_JNI", "-I", os.path.join(ROOT, "tests", "jni_stub"), src],
                       capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr[-3000:]
    text = open(src).read()
    for name in ("batchRowsAsync", "batchRowsWithPartitionAsync"):
        assert f"Java_com_linkedin_spark_datasources_tfrecord_TfrGpu_{name}(" in text
