"""CPU tests of the UnsafeRow builder (oracle/unsaferow.py) that the row-encode tests and tools/quick_rows_encode.py use:
known-answer layouts derived by hand from Spark's UnsafeRow / UnsafeArrayData format."""
import numpy as np

from oracle import unsaferow as U
from spark_tfrecord_b200.sqltypes import *  # noqa


def h(s: str) -> bytes:
    return bytes.fromhex(s.replace(" ", ""))


def test_golden_example_row():
    sch = StructType([StructField("LongLabel", LongType()), StructField("FloatLabel", FloatType()), StructField("StrLabel", StringType())])
    got = U.unsafe_row(sch, (23, 10.0, "r1"))
    assert len(got) == 40
    assert got == h("00" * 8 + "17" + "00" * 7 + "00002041" + "00" * 4 + "0200000020000000" + "7231" + "00" * 6)


def test_long_array_at_offset_16():
    got = U.unsafe_row(StructType([StructField("a", ArrayType(LongType()))]), ([1, 2],))
    assert got[8:16] == h("2000000010000000")
    arr = got[16:]
    assert len(arr) == 32 and arr == h("0200000000000000" + "00" * 8 + "0100000000000000" + "0200000000000000")


def test_int_array_padding_and_empty_array():
    arr = U.unsafe_array(TFR_T_INT32, 1, [1, 2, 3])
    assert len(arr) == 32 and arr == h("0300000000000000" + "00" * 8 + "01000000" "02000000" "03000000" + "00000000")
    assert U.unsafe_array(TFR_T_INT64, 1, []) == h("00" * 8)


def test_string_array_element_slot():
    arr = U.unsafe_array(TFR_T_STRING, 1, ["a"])
    assert arr[16:24] == ((24 << 32) | 1).to_bytes(8, "little")
    assert arr[24:] == b"a" + b"\0" * 7


def test_nulls_and_garbage():
    sch = StructType([StructField("x", LongType()), StructField("v", ArrayType(IntegerType()))])
    row = U.unsafe_row(sch, (None, [7, None, 9]))
    assert row[0] == 1 and row[8:16] == b"\0" * 8                       # null field: bit 0, zero slot
    arr = row[24:]
    assert arr[8] == 0b10 and arr[16 + 4:16 + 8] == b"\0" * 4            # null element: bit 1, zero slot
    g = U.unsafe_row(sch, (None, [7, None, 9]), garbage=True, seed=3)
    assert g[:24 + 20] == row[:24 + 20] and g[24 + 20:24 + 24] != b"\0" * 4 and g[24 + 24:] == row[24 + 24:]


def test_nested_array_and_decimal():
    sch = StructType([StructField("d", DecimalType()), StructField("aa", ArrayType(ArrayType(StringType())))])
    row = U.unsafe_row(sch, (-5, [["ab"], []]))
    assert row[8:16] == (-5 & (2**64 - 1)).to_bytes(8, "little")
    off, size = int.from_bytes(row[20:24], "little"), int.from_bytes(row[16:20], "little")
    outer = row[off:off + size]
    assert int.from_bytes(outer[:8], "little") == 2
    s0 = int.from_bytes(outer[16:24], "little")
    inner = outer[s0 >> 32:(s0 >> 32) + (s0 & 0xFFFFFFFF)]
    assert inner == U.unsafe_array(TFR_T_STRING, 1, ["ab"])


def test_vectorised_cfg2_rows_match_the_row_builder():
    from oracle.corpus import cfg2_columns
    from spark_tfrecord_b200 import _cabi as A
    sch, cols = cfg2_columns(40, seed=4)
    data, offs = U.cfg2_rows(cols)
    assert offs[1] == 1544
    rows = [tuple(c.get(r) for c in cols) for r in range(40)]
    want, woffs = U.unsafe_rows(sch, rows)
    assert np.array_equal(offs, woffs) and np.array_equal(data, want)
