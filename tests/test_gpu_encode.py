"""GPU parity tests for the encode path: tfr_encode output must be byte-identical to the oracle writer
(restating TFRecordSerializer + protobuf-java toByteArray + TFRecordWriter), and decode(encode(x)) == x."""
import numpy as np
import pytest

from util import assert_columns_equal
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def gpu_encode(native, schema, cols, record_type=0):
    enc = native.Encoder(schema, record_type)
    try:
        return enc.encode(cols)
    finally:
        enc.close()


def _diff(a: bytes, b: bytes):
    if a == b:
        return None
    n = min(len(a), len(b))
    x = np.frombuffer(a[:n], np.uint8) != np.frombuffer(b[:n], np.uint8)
    pos = int(np.argmax(x)) if x.any() else n
    return f"len {len(a)} vs {len(b)}; first diff at {pos}: {a[max(0,pos-8):pos+8].hex()} vs {b[max(0,pos-8):pos+8].hex()}"


def _check(native, oracle, schema, cols, record_type=0):
    want, rc, _ = oracle.encode(cols, schema, record_type)
    assert rc == 0
    got = gpu_encode(native, schema, cols, record_type)
    assert _diff(got, want) is None, _diff(got, want)
    # and the decoder reads it back bit-exactly (CRC verified)
    dec = native.Decoder(schema, record_type)
    batch, used = dec.decode(got)
    assert batch.info["error_code"] == 0 and used == len(got)
    back = batch.to_host()
    batch.release()
    dec.close()
    return got, back


def test_golden_example_bytes(native, oracle):
    from oracle import pyref
    sch = StructType([StructField("LongLabel", LongType()), StructField("FloatLabel", FloatType()), StructField("StrLabel", StringType())])
    cols = A.columns_from_rows(sch, [(23, 10.0, "r1")])
    got = gpu_encode(native, sch, cols)
    want = bytes.fromhex("0a40" "0a12" "0a094c6f6e674c6162656c" "1205" "1a03" "0a01" "17" "0a16" "0a0a466c6f61744c6162656c" "1208" "1206"
                         "0a04" "00002041" "0a12" "0a085374724c6162656c" "1206" "0a04" "0a02" "7231")
    assert got == pyref.frame(want)


def test_reference_io_suite_rows(native, oracle):
    import cases as CS
    for c in CS.reference_cases():
        if c.name == "ref_io_suite_example":
            rows = c.rows
            cols = A.columns_from_rows(c.schema, [tuple(r) for r in rows])
            got, back = _check(native, oracle, c.schema, cols)
            assert got == c.data()        # identical to pyref/upb's serialisation in schema order
        if c.name == "ref_io_suite_sequence":
            cols = A.columns_from_rows(c.schema, [tuple(r) for r in c.rows])
            got, back = _check(native, oracle, c.schema, cols, TFR_RT_SEQUENCE_EXAMPLE)
            assert got == c.data()


def test_cfg1(native, oracle):
    from oracle.corpus import cfg1_columns
    sch, cols = cfg1_columns(10_000, seed=1234)
    got, back = _check(native, oracle, sch, cols)
    assert_columns_equal(back, cols, sch.names, "cfg1 encode->decode")


@pytest.mark.parametrize("n", [1, 31, 5000])
def test_cfg2(native, oracle, n):
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(n, seed=3 + n)
    got, back = _check(native, oracle, sch, cols)
    assert_columns_equal(back, cols, sch.names, "cfg2 encode->decode")


def test_mixed_with_nulls(native, oracle):
    from oracle.corpus import mixed_columns
    sch, cols = mixed_columns(3000, seed=21)
    got, back = _check(native, oracle, sch, cols)
    assert_columns_equal(back, cols, sch.names, "mixed encode->decode")


def test_cfg4_sequence_example(native, oracle):
    from oracle.corpus import cfg4_columns
    sch, cols = cfg4_columns(800, seed=78)
    got, back = _check(native, oracle, sch, cols, TFR_RT_SEQUENCE_EXAMPLE)
    assert_columns_equal(back, cols, sch.names, "cfg4 encode->decode")


def test_bytearray(native, oracle):
    rng = np.random.default_rng(5)
    rows = [(rng.integers(0, 256, int(s), dtype=np.uint8).tobytes(),) for s in [0, 1, 2, 3, 4, 5, 127, 128, 129, 4096, 100000] + list(rng.integers(0, 2000, 300))]
    sch = byte_array_schema()
    cols = A.columns_from_rows(sch, rows)
    _check(native, oracle, sch, cols, TFR_RT_BYTE_ARRAY)


def test_double_narrowing_and_int_widening(native, oracle):
    """Double -> FloatList via toFloat (RNE, overflow to inf, NaN kept quiet); Integer sign-extends"""
    d = np.array([0.1, 1e40, -1e40, 1e-50, 3.4028235677973366e38, 1.0000000596046448, float("nan"), -0.0, 16777217.0, 2.5], dtype=np.float64)
    nan_payload = np.array([0x7FF8000012345678, 0xFFF0000000000001, 0x7FF4000000000000], dtype=np.uint64).view(np.float64)
    d = np.concatenate([d, nan_payload])
    i = np.array([0, -1, 2**31 - 1, -2**31, 127, 128, -129] + [5] * (len(d) - 7), dtype=np.int32)
    n = len(d)
    sch = StructType([StructField("d", DoubleType()), StructField("i", IntegerType()), StructField("da", ArrayType(DoubleType()))])
    full = np.full((n + 7) // 8, 0xFF, np.uint8)
    cols = [A.HostColumn(TFR_T_FLOAT64, 0, n, full, [], d), A.HostColumn(TFR_T_INT32, 0, n, full, [], i),
            A.HostColumn(TFR_T_FLOAT64, 1, n, full, [np.arange(n + 1, dtype=np.int32)], d)]
    want, rc, _ = oracle.encode(cols, sch)
    got = gpu_encode(native, sch, cols)
    assert _diff(got, want) is None, _diff(got, want)


def test_nulls_omitted_and_wrappers(native, oracle):
    from oracle import pyref
    sch = StructType([StructField("NullLabel", ArrayType(FloatType()), True), StructField("FloatArrayLabel", ArrayType(FloatType()))])
    cols = A.columns_from_rows(sch, [(None, [2.5, 5.0]), (None, None), ([], [])])
    _check(native, oracle, sch, cols)
    _check(native, oracle, sch, cols, TFR_RT_SEQUENCE_EXAMPLE)
    got = gpu_encode(native, sch, A.columns_from_rows(sch, [(None, None)]))
    assert got == pyref.frame(bytes.fromhex("0a00"))
    got = gpu_encode(native, sch, A.columns_from_rows(sch, [(None, None)]), TFR_RT_SEQUENCE_EXAMPLE)
    assert got == pyref.frame(bytes.fromhex("0a001200"))


def test_null_in_nonnullable_is_npe(native, oracle):
    # T/TFRecordSerializerTest.scala:229-245
    sch = StructType([StructField("ok", LongType()), StructField("NonNullLabel", ArrayType(FloatType()), nullable=False)])
    cols = A.columns_from_rows(sch, [(1, [1.0]), (2, [2.0]), (3, None), (4, None)])
    for rt in (TFR_RT_EXAMPLE, TFR_RT_SEQUENCE_EXAMPLE):
        with pytest.raises(native.NullPointerException) as ei:
            gpu_encode(native, sch, cols, rt)
        assert ei.value.row == 2
        _, rc, er = oracle.encode(cols, sch, rt)
        assert rc == A.TFR_E_NULL_IN_NONNULL and er == 2


def test_unsupported_types_throw_at_construction(native):
    # T/TFRecordSerializerTest.scala:290-299 (+ the decoder's runtime equivalent)
    with pytest.raises(native.UnsupportedTypeException):
        native.Encoder(StructType([StructField("TimestampLabel", TimestampType())]))
    with pytest.raises(native.UnsupportedTypeException):
        native.Decoder(StructType([StructField("MapLabel1", TimestampType())]))
    with pytest.raises(native.UnsupportedTypeException):
        native.Encoder(StructType([StructField("x", ArrayType(ArrayType(LongType())))]), TFR_RT_EXAMPLE)
    with pytest.raises(native.IllegalArgumentException):
        native.Schema(StructType([StructField("x", LongType())]), 7)


def test_many_fields_more_than_a_warp(native, oracle):
    rng = np.random.default_rng(1)
    nfld, n = 100, 200
    sch = StructType([StructField(f"c{i:03d}", LongType() if i % 3 else ArrayType(StringType())) for i in range(nfld)])
    rows = []
    for r in range(n):
        row = []
        for i in range(nfld):
            if rng.random() < 0.1:
                row.append(None)
            elif i % 3:
                row.append(int(rng.integers(-2**40, 2**40)))
            else:
                row.append(["s%d" % int(x) for x in rng.integers(0, 1000, int(rng.integers(0, 4)))])
        rows.append(tuple(row))
    cols = A.columns_from_rows(sch, rows)
    got, back = _check(native, oracle, sch, cols)
    assert_columns_equal(back, cols, sch.names, "100 fields")


def test_tile_emit_shapes(native, oracle):
    """the tile emit kernel: row counts around the 32-row tile, nulls, empty lists and strings, one long row among
    short ones, every Int64 varint width; and the same bytes through the general kernel"""
    import os
    rng = np.random.default_rng(5)
    sch = StructType([StructField("a", LongType()), StructField("i", IntegerType()), StructField("f", ArrayType(FloatType())),
                      StructField("d", DoubleType()), StructField("s", StringType()), StructField("b", ArrayType(BinaryType())),
                      StructField("v", ArrayType(LongType()))])
    def row(i):
        width = i % 11
        a = None if i % 13 == 5 else (int(rng.integers(0, 100)) if width == 0 else (-(i + 1) if width == 10 else int(1 << (7 * width - 1)) + i))
        f = None if i % 17 == 3 else [float(x) for x in rng.standard_normal(i % 9).astype(np.float32)]
        s = None if i % 19 == 7 else "".join(chr(97 + (i + k) % 26) for k in range(i % 31))
        b = [rng.integers(0, 256, (i + k) % 7, dtype=np.uint8).tobytes() for k in range(i % 4)]
        v = [int(x) for x in rng.integers(-2**62, 2**62, i % 5)]
        return (a, int(rng.integers(-2**31, 2**31)), f, float(rng.standard_normal()), s, b, v)
    for n in (1, 31, 32, 33, 64, 257):
        rows = [row(i) for i in range(n)]
        if n == 257:
            rows[100] = (1, 2, [1.0] * 900, 3.0, "y" * 2500, [b"z" * 700], list(range(200)))
        cols = A.columns_from_rows(sch, rows)
        want, rc, _ = oracle.encode(cols, sch, 0)
        assert rc == 0
        got = gpu_encode(native, sch, cols, 0)
        assert got == want, _diff(got, want)
        os.environ["TFR_DISABLE_FAST"] = "1"
        try:
            got2 = gpu_encode(native, sch, cols, 0)
        finally:
            del os.environ["TFR_DISABLE_FAST"]
        assert got2 == want, _diff(got2, want)


def test_encoder_reused_across_row_sizes(native, oracle):
    """One encoder, many calls: row counts that fill no, one or many tiles, other varint widths, ragged rows with nulls, a
    batch with one row far larger than the ones before: same bytes as the oracle; a null in a non-nullable column is
    reported at the same row, and the encoder goes on encoding."""
    from oracle.corpus import cfg2_columns, mixed_columns
    rng = np.random.default_rng(9)
    sch, cols = cfg2_columns(3000, seed=77)
    want, rc, _ = oracle.encode(cols, sch)
    enc = native.Encoder(sch, 0)
    try:
        for _ in range(3):
            assert enc.encode(cols) == want
        sch2, cols2 = cfg2_columns(1, seed=78)                     # a single row: one partial tile
        want2, _, _ = oracle.encode(cols2, sch2)
        assert enc.encode(cols2) == want2
        sch3, cols3 = cfg2_columns(4097, seed=79, small_ints=True) # other varint widths, 129 tiles
        want3, _, _ = oracle.encode(cols3, sch3)
        assert enc.encode(cols3) == want3
    finally:
        enc.close()
    # ragged rows, nulls, strings; then one row far larger than anything seen before
    schm = StructType([StructField("a", LongType()), StructField("s", StringType()), StructField("v", ArrayType(LongType())),
                       StructField("f", ArrayType(FloatType())), StructField("b", ArrayType(BinaryType()))])
    def rows(n, big=None):
        out = []
        for i in range(n):
            out.append((None if i % 7 == 3 else int(rng.integers(-2**62, 2**62)), None if i % 5 == 1 else "s" * (i % 40),
                        [int(x) for x in rng.integers(-1000, 1000, i % 6)], [float(x) for x in rng.standard_normal(i % 4).astype(np.float32)],
                        [bytes(rng.integers(0, 256, (i + k) % 9, dtype=np.uint8)) for k in range(i % 3)]))
        if big is not None:
            out[big] = (5, "y" * 3000, list(range(500)), [1.5] * 700, [b"z" * 900])
        return out
    enc = native.Encoder(schm, 0)
    try:
        for data in (rows(500), rows(500), rows(777, big=300), rows(777, big=5), rows(64)):
            c = A.columns_from_rows(schm, data)
            w, rc, _ = oracle.encode(c, schm)
            assert rc == 0
            g = enc.encode(c)
            assert g == w, _diff(g, w)
    finally:
        enc.close()
    # NullPointerException on an encoder that has encoded before
    schn = StructType([StructField("ok", LongType()), StructField("NonNullLabel", ArrayType(FloatType()), nullable=False)])
    good = A.columns_from_rows(schn, [(i, [1.0 * i]) for i in range(100)])
    bad = A.columns_from_rows(schn, [(i, None if i in (41, 77) else [1.0 * i]) for i in range(100)])
    enc = native.Encoder(schn, 0)
    try:
        w, _, _ = oracle.encode(good, schn)
        assert enc.encode(good) == w and enc.encode(good) == w
        with pytest.raises(native.NullPointerException) as ei:
            enc.encode(bad)
        assert ei.value.row == 41
        assert enc.encode(good) == w
    finally:
        enc.close()
