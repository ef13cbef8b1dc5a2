"""CPU check of oracle.unsaferow's builder by an independent reader (tests/unsafe_row_reader.py): every row built from
random schemas of all non-decimal types, nulls, empty and nested arrays parses back to the values it was built from."""
import numpy as np
import pytest

from oracle import unsaferow as U
from spark_tfrecord_b200.sqltypes import *  # noqa
import unsafe_row_reader as R


def _rand_schema(rng):
    from test_gpu_fuzz import _schema
    return _schema(rng, seq=bool(rng.random() < 0.5))


@pytest.mark.parametrize("seed", range(24))
def test_reader_parses_builder_rows(seed):
    rng = np.random.default_rng(seed)
    sch, gens = _rand_schema(rng)
    if seed % 4 == 0:                                       # NullType and a 64+ field row: two null words
        sch = StructType(list(sch) + [StructField("nul", NullType())] + [StructField(f"x{i}", IntegerType()) for i in range(60)])
        gens = list(gens) + [lambda r: None] + [lambda r: int(r.integers(-2**31, 2**31)) for _ in range(60)]
    rows = [tuple(g(rng) for g in gens) for _ in range(40)]
    data, offs = U.unsafe_rows(sch, rows)
    assert offs[0] == 0 and all(o % 8 == 0 for o in offs)
    got = R.read_rows(sch, data, offs)
    for r, (g, w) in enumerate(zip(got, rows)):
        assert g == R.normalise(sch, w), (r, g, w)


def test_reader_float_bits_and_layout():
    sch = StructType([StructField("f", FloatType()), StructField("d", DoubleType()), StructField("s", StringType()),
                      StructField("a", ArrayType(FloatType()))])
    nan = np.array([0x7FC12345], np.uint32).view(np.float32)[0]
    rows = [(nan, np.float64(-0.0), "", [np.float32(-0.0), nan, np.float32(1.5)]), (None, None, None, None), (1.0, 2.0, "é", [])]
    data, offs = U.unsafe_rows(sch, rows)
    got = R.read_rows(sch, data, offs)
    assert got[0][0] == 0x7FC12345 and got[0][1] == 1 << 63 and got[0][2] == b"" and got[0][3] == [0x80000000, 0x7FC12345, 0x3FC00000]
    assert got[1] == (None, None, None, None)
    assert got[2][3] == [] and got[2][2] == "é".encode()
    # a differing element is reported by row and field
    d2 = data.copy()
    d2[int(offs[2]) + 8] ^= 1                               # the float slot of row 2
    assert R.first_diff(sch, d2, offs, data, offs).startswith("row 2 field 0")


def test_reader_rejects_broken_rows():
    sch = StructType([StructField("s", StringType())])
    data, offs = U.unsafe_rows(sch, [("abc",)])
    bad = data.copy()
    bad[8 + 3 + 8] = 1                                      # a padding byte after "abc"
    with pytest.raises(ValueError):
        R.read_rows(sch, bad, offs)
