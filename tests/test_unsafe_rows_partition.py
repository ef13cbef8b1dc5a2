"""CPU test of tests/partition_rows.py, the writer of joined data + partition UnsafeRows the GPU rows are compared with:
pinned against hand-derived layouts of each partition type (UnsafeRowWriter's rules restated in include/tfrgpu.h)."""
import struct

import numpy as np
import pytest

import partition_rows as P
from oracle import unsaferow as U
from spark_tfrecord_b200.sqltypes import LongType, StringType, StructField, StructType


def h(s: str) -> bytes:
    return bytes.fromhex(s.replace(" ", ""))


Z8 = "00" * 8
NULL0 = "01" + "00" * 7                                     # null bitset word with bit 0 set

# (type, value, the partition row of P = [type]: null word, slot, variable region)
CASES = [
    ("boolean", True, Z8 + "01 00 00 00 00 00 00 00"),
    ("boolean", None, NULL0 + Z8),
    ("byte", -1, Z8 + "ff 00 00 00 00 00 00 00"),
    ("byte", None, NULL0 + Z8),
    ("short", -2, Z8 + "fe ff 00 00 00 00 00 00"),
    ("short", None, NULL0 + Z8),
    ("int", 7, Z8 + "07 00 00 00 00 00 00 00"),
    ("int", -1, Z8 + "ff ff ff ff 00 00 00 00"),
    ("int", None, NULL0 + Z8),
    ("long", -1, Z8 + "ff" * 8),
    ("long", None, NULL0 + Z8),
    ("float", 1.0, Z8 + "00 00 80 3f 00 00 00 00"),
    ("float", None, NULL0 + Z8),
    ("double", 1.0, Z8 + "00 00 00 00 00 00 f0 3f"),
    ("double", None, NULL0 + Z8),
    ("date", 19000, Z8 + "38 4a 00 00 00 00 00 00"),           # 2022-01-08, int days
    ("date", None, NULL0 + Z8),
    ("timestamp", 1, Z8 + "01 00 00 00 00 00 00 00"),          # long microseconds
    ("timestamp", None, NULL0 + Z8),
    ("string", "ab", Z8 + "02 00 00 00 10 00 00 00" + "61 62 00 00 00 00 00 00"),
    ("string", "", Z8 + "00 00 00 00 10 00 00 00"),            # empty, not null: offset 16, size 0
    ("string", None, NULL0 + Z8),
    ("binary", bytes(range(1, 10)), Z8 + "09 00 00 00 10 00 00 00" + "01 02 03 04 05 06 07 08 09" + "00" * 7),
    ("binary", None, NULL0 + Z8),
    (("decimal", 10, 2), 12345, Z8 + "39 30 00 00 00 00 00 00"),  # precision <= 18: the unscaled long in the slot
    (("decimal", 10, 2), None, NULL0 + Z8),
    # precision > 18: 16 reserved zero bytes, BigInteger.toByteArray() at their start, the slot holds its length
    (("decimal", 38, 6), 10 ** 20, Z8 + "09 00 00 00 10 00 00 00" + "05 6b c7 5e 2d 63 10 00 00" + "00" * 7),
    (("decimal", 38, 6), -10 ** 20, Z8 + "09 00 00 00 10 00 00 00" + "fa 94 38 a1 d2 9c f0 00 00" + "00" * 7),
    (("decimal", 38, 6), 0, Z8 + "01 00 00 00 10 00 00 00" + "00" * 16),
    (("decimal", 38, 6), -1, Z8 + "01 00 00 00 10 00 00 00" + "ff" + "00" * 15),
    (("decimal", 38, 6), None, NULL0 + "00 00 00 00 10 00 00 00" + "00" * 16),   # bit set, offset kept, size 0
]


@pytest.mark.parametrize("t,v,want", CASES, ids=[f"{c[0]}-{c[1]!r:.12}" for c in CASES])
def test_partition_row_layout(t, v, want):
    assert P.partition_row([t], [v]) == h(want)


def test_var_flags():
    assert P.var_flags(P.PART_TYPES) == bytes([0] * 9 + [1, 1, 0, 1])


def test_big_decimal_bytes():
    assert P.big_decimal_bytes(0) == b"\0" and P.big_decimal_bytes(127) == b"\x7f" and P.big_decimal_bytes(128) == b"\0\x80"
    assert P.big_decimal_bytes(-128) == b"\x80" and P.big_decimal_bytes(-129) == b"\xff\x7f"
    assert P.big_decimal_bytes(10 ** 38 - 1) == (10 ** 38 - 1).to_bytes(16, "big")


def test_no_partition_fields_is_the_data_row():
    sch = StructType([StructField("a", LongType()), StructField("s", StringType())])
    for row in [(1, "xyz"), (None, ""), (5, None)]:
        assert P.joined_row(sch, row, [], []) == U.unsafe_row(sch, row)


def test_joined_row_two_null_words():
    """nd = 63 longs + np = 2 (int, string): 65 fields, the bitset grows to two words; data field 62 is null"""
    sch = StructType([StructField(f"l{i}", LongType()) for i in range(63)])
    row = [i * 3 for i in range(62)] + [None]
    got = P.joined_row(sch, row, ["int", "string"], [5, "x"])
    fixed = 8 * (2 + 65)                                     # 536
    want = bytearray(fixed + 8)
    want[7] = 0x40                                           # bit 62 of word 0
    for i in range(62):
        want[16 + 8 * i:24 + 8 * i] = struct.pack("<q", i * 3)
    want[16 + 8 * 63:24 + 8 * 63] = struct.pack("<q", 5)
    want[16 + 8 * 64:24 + 8 * 64] = struct.pack("<Q", (fixed << 32) | 1)
    want[fixed] = ord("x")
    assert got == bytes(want)
    # the partition string null: bit 64 = bit 0 of word 1, slot zero, no variable bytes
    got = P.joined_row(sch, row, ["int", "string"], [5, None])
    want = want[:fixed]
    want[8] = 0x01
    want[16 + 8 * 64:24 + 8 * 64] = bytes(8)
    assert got == bytes(want)


def test_cfg2_joined_rows_match_the_writer():
    from oracle.corpus import cfg2_columns
    from test_gpu_encode_rows import rows_of
    sch, cols = cfg2_columns(5, seed=3)
    pt, pv = ["string", "int", ("decimal", 38, 6)], ["2024-01-01", 42, None]
    vr, vo = P.cfg2_joined_rows(cols, pt, pv)
    wr, wo = P.joined_rows(sch, rows_of(cols, 5), pt, pv)
    assert np.array_equal(vo, wo) and np.array_equal(vr, wr)
