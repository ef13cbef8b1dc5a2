"""GPU tests of tfr_encode_rows: Spark UnsafeRows -> framed records.  Every batch is compared byte for byte with tfr_encode
of the same rows given as columns and with the oracle writer, then decoded back by the decoder (CRC verified).
Reference semantics: M/TFRecordSerializer.scala:20-60,68-207, M/TFRecordOutputWriter.scala:26-38."""
import numpy as np
import pytest

from oracle import unsaferow as U
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def _diff(a: bytes, b: bytes):
    if a == b:
        return None
    n = min(len(a), len(b))
    x = np.frombuffer(a[:n], np.uint8) != np.frombuffer(b[:n], np.uint8)
    pos = int(np.argmax(x)) if x.any() else n
    return f"len {len(a)} vs {len(b)}; first diff at {pos}"


def rows_of(cols, n):
    """Python rows of HostColumns, fixed-width leaves as numpy scalars (exact float bits)"""
    def cell(c, r):
        if c.elem_type in (TFR_T_STRING, TFR_T_BINARY) or not c.valid(r):
            return c.get(r)
        if c.depth == 0:
            return c.values[r]
        o0 = c.offsets[0]
        if c.depth == 1:
            return list(c.values[o0[r]:o0[r + 1]])
        o1 = c.offsets[1]
        return [list(c.values[o1[s]:o1[s + 1]]) for s in range(o0[r], o0[r + 1])]
    return [tuple(cell(c, r) for c in cols) for r in range(n)]


def check(native, oracle, sch, cols, rt=0, data=None, decode=True):
    """rows (built from cols unless given) through tfr_encode_rows == tfr_encode(cols) == oracle; decoded back"""
    want, rc, _ = oracle.encode(cols, sch, rt)
    assert rc == 0
    if data is None:
        data = U.unsafe_rows(sch, rows_of(cols, cols[0].n_rows))
    enc = native.Encoder(sch, rt)
    try:
        assert enc.encode(cols) == want
        enc.encode_rows(*data)
        got = enc.result_host()
    finally:
        enc.close()
    assert got == want, _diff(got, want)
    if decode:
        dec = native.Decoder(sch, rt)
        b, used = dec.decode(got)
        assert b.info["error_code"] == 0 and used == len(got)
        b.release()
        dec.close()
    return got


def rows_error(native, sch, data, offs, rt=0):
    enc = native.Encoder(sch, rt)
    try:
        with pytest.raises(native.TfrError) as ei:
            enc.encode_rows(data, offs)
        return ei.value.code, ei.value.row
    finally:
        enc.close()


def test_golden_example(native, oracle):
    from oracle import pyref
    sch = StructType([StructField("LongLabel", LongType()), StructField("FloatLabel", FloatType()), StructField("StrLabel", StringType())])
    got = check(native, oracle, sch, A.columns_from_rows(sch, [(23, 10.0, "r1")]))
    payload = bytes.fromhex("0a40" "0a12" "0a094c6f6e674c6162656c" "1205" "1a03" "0a01" "17" "0a16" "0a0a466c6f61744c6162656c" "1208" "1206"
                            "0a04" "00002041" "0a12" "0a085374724c6162656c" "1206" "0a04" "0a02" "7231")
    assert len(payload) == 66 and got == pyref.frame(payload)


def _scale0(sch, rows):
    """an UnsafeRow holds a DecimalType(10, 0) value as its unscaled long: the suite's 1.1 is 1 there.  -> (rows with the
    unscaled ints, rows with what the writer makes of them as the column path's float64)"""
    dec = [lower_type(f.dataType)[0] == TFR_T_DECIMAL for f in sch]
    def conv(v, d, as_float):
        if v is None or not d:
            return v
        if isinstance(v, list):
            return [conv(x, d, as_float) for x in v]
        i = int(round(v))
        return float(np.float32(i)) if as_float else i
    return ([tuple(conv(v, d, False) for v, d in zip(r, dec)) for r in rows],
            [tuple(conv(v, d, True) for v, d in zip(r, dec)) for r in rows], any(dec))


def test_reference_io_suite_rows(native, oracle):
    import cases as CS
    for c in CS.reference_cases():
        if c.name in ("ref_io_suite_example", "ref_io_suite_sequence"):
            rt = TFR_RT_SEQUENCE_EXAMPLE if c.name.endswith("sequence") else TFR_RT_EXAMPLE
            rows, as_cols, has_dec = _scale0(c.schema, [tuple(r) for r in c.rows])
            got = check(native, oracle, c.schema, A.columns_from_rows(c.schema, as_cols, rt), rt, data=U.unsafe_rows(c.schema, rows))
            if not has_dec:
                assert got == c.data()


def test_cfg1(native, oracle):
    from oracle.corpus import cfg1_columns
    sch, cols = cfg1_columns(10_000, seed=1234)
    check(native, oracle, sch, cols)


@pytest.mark.parametrize("n", [1, 31, 5000, 250_000])
def test_cfg2(native, oracle, n):
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(n, seed=3 + n)
    check(native, oracle, sch, cols, data=U.cfg2_rows(cols), decode=n < 100_000)


def test_mixed_columns(native, oracle):
    from oracle.corpus import mixed_columns
    sch, cols = mixed_columns(3000, seed=21)
    check(native, oracle, sch, cols)


def test_cfg4_sequence_example(native, oracle):
    from oracle.corpus import cfg4_columns
    sch, cols = cfg4_columns(800, seed=78)
    check(native, oracle, sch, cols, TFR_RT_SEQUENCE_EXAMPLE)


def test_bytearray(native, oracle):
    rng = np.random.default_rng(5)
    rows = [(rng.integers(0, 256, int(s), dtype=np.uint8).tobytes(),) for s in [0, 1, 2, 3, 4, 5, 127, 128, 129, 4096, 100000] + list(rng.integers(0, 2000, 300))]
    sch = byte_array_schema()
    check(native, oracle, sch, A.columns_from_rows(sch, rows), TFR_RT_BYTE_ARRAY)


_ROW_LEAVES = [("i", IntegerType), ("l", LongType), ("f", FloatType), ("d", DoubleType), ("s", StringType), ("b", BinaryType),
               ("m", DecimalType)]


def _row_leaf(r, kind, null_elem=False, garbage=False):
    """-> (the value in the UnsafeRow, the value the column path is given for it)"""
    from test_gpu_fuzz import _leaf
    if null_elem:                                  # a null element of a numeric array: its slot's bits are encoded
        if not garbage:
            g = 0.0 if kind in ("f", "d") else 0
        elif kind == "i":
            g = int(r.integers(-2**31, 2**31))
        elif kind == "l":
            g = int(r.integers(-2**63, 2**63 - 1))
        else:
            g = float(np.float32(r.standard_normal()))
        return U.NullElem(g), g
    if kind == "m":
        v = int(r.integers(-2**63, 2**63 - 1)) if r.random() < 0.5 else int(r.integers(-1000, 1000))
        return v, float(np.float32(np.int64(v)))
    v = _leaf(r, kind)
    return v, v


def _row_schema(rng, seq, garbage):
    """random schemas over every leaf type (DecimalType included): scalars, 1-D and (SequenceExample) 2-D arrays, nullable
    and required fields, null fields, and null elements in numeric arrays (zero slots, or other bits with `garbage`)"""
    k = int(rng.integers(1, 15))
    fields, gens = [], []
    for j in range(k):
        kind, dt = _ROW_LEAVES[int(rng.integers(0, len(_ROW_LEAVES)))]
        depth = 2 if seq and rng.random() < 0.4 else (1 if rng.random() < 0.45 else 0)
        nullable = depth == 2 or rng.random() < 0.7
        null_frac = float(rng.choice([0.0, 0.1, 0.5])) if nullable else 0.0
        elem_null = 0.15 if kind in ("i", "l", "f", "d") and rng.random() < 0.6 else 0.0
        t = dt()
        for _ in range(depth):
            t = ArrayType(t)
        fields.append(StructField(f"c{j}_{kind}{depth}", t, nullable))

        def gen(r, kind=kind, depth=depth, null_frac=null_frac, elem_null=elem_null):
            if r.random() < null_frac:
                return None, None
            def arr():
                pairs = [_row_leaf(r, kind, r.random() < elem_null, garbage) for _ in range(int(r.integers(0, 7)))]
                return [a for a, _ in pairs], [b for _, b in pairs]
            if depth == 0:
                return _row_leaf(r, kind)
            if depth == 1:
                return arr()
            steps = [arr() for _ in range(int(r.integers(0, 5)))]
            return [a for a, _ in steps], [b for _, b in steps]
        gens.append(gen)
    return StructType(fields), gens


@pytest.mark.parametrize("seed", range(80))
def test_random_schemas(native, oracle, seed):
    """every leaf type, scalar, 1-D and (SequenceExample) 2-D, nullable and required, null fields and null numeric elements"""
    rt = seed % 2
    garbage = (seed // 2) % 2 == 1
    rng = np.random.default_rng(40000 + seed)
    sch, gens = _row_schema(rng, bool(rt), garbage)
    n = int(rng.choice([1, 33, 300, 1200]))
    r = np.random.default_rng(seed)
    pairs = [[g(r) for g in gens] for _ in range(n)]
    rows = [tuple(a for a, _ in p) for p in pairs]
    as_cols = [tuple(b for _, b in p) for p in pairs]
    check(native, oracle, sch, A.columns_from_rows(sch, as_cols, rt), rt, data=U.unsafe_rows(sch, rows))


@pytest.mark.parametrize("rt", [TFR_RT_BYTE_ARRAY, TFR_RT_EXAMPLE])
def test_offsets_down_and_up_are_invalid_arg(native, oracle, rt):
    """offsets [0, L, 0, L, ...]: every second row runs backwards, the rows between them are well-formed and overlap, so
    their totals exceed anything sized from the input.  TFR_E_INVALID_ARG at row 1, and the encoder goes on working."""
    rng = np.random.default_rng(12)
    payload = rng.integers(0, 256, 4000, dtype=np.uint8).tobytes()
    if rt == TFR_RT_BYTE_ARRAY:
        sch, row = byte_array_schema(), (payload,)
    else:
        sch, row = StructType([StructField("id", LongType()), StructField("b", BinaryType()), StructField("v", ArrayType(FloatType()))]), \
            (7, payload, [1.5] * 300)
    data, offs1 = U.unsafe_rows(sch, [row])
    L = int(offs1[1])
    offs = np.array([0 if i % 2 == 0 else L for i in range(1000)], dtype=np.int32)      # 999 rows, offs[999] = L
    enc = native.Encoder(sch, rt)
    try:
        for _ in range(2):
            with pytest.raises(native.TfrError) as ei:
                enc.encode_rows(data, offs)
            assert (ei.value.code, ei.value.row) == (A.TFR_E_INVALID_ARG, 1)
        good = [row] * 5
        want, rc, _ = oracle.encode(A.columns_from_rows(sch, good, rt), sch, rt)
        enc.encode_rows(*U.unsafe_rows(sch, good))
        assert rc == 0 and enc.result_host() == want
    finally:
        enc.close()


def test_decimal_rounds_int64_to_float_once(native, oracle):
    """BigDecimal(v, 0).floatValue: one round to nearest even from the int64, never through a double"""
    vals = [0, 1, -1, 2**24 - 1, 2**24, 2**24 + 1, -(2**24 + 1), 2**24 + 3, 2**53 - 1, 2**53 + 1, -(2**53 + 1), 2**60 + 2**36 + 1,
            -(2**60 + 2**36 + 1), 2**63 - 1, -2**63, 12345678901234567]
    rng = np.random.default_rng(3)
    vals += [int(x) for x in rng.integers(-2**63, 2**63 - 1, 200, dtype=np.int64, endpoint=True)]
    as_float = [float(x) for x in np.array(vals, dtype=np.int64).astype(np.float32)]
    sch = StructType([StructField("d", DecimalType()), StructField("da", ArrayType(DecimalType()))])
    rows = [(v, [v, -v if v != -2**63 else v]) for v in vals]
    want_rows = [(f, [f, float(np.float32(np.int64(-v if v != -2**63 else v)))]) for v, f in zip(vals, as_float)]
    cols = A.columns_from_rows(sch, want_rows)
    check(native, oracle, sch, cols, data=U.unsafe_rows(sch, rows))


def test_null_numeric_elements_keep_their_bits(native, oracle):
    sch = StructType([StructField("i", ArrayType(IntegerType())), StructField("l", ArrayType(LongType())),
                      StructField("f", ArrayType(FloatType())), StructField("d", ArrayType(DoubleType()))])
    rows = [([1, None, 3], [None, 5], [None, 1.5], [2.5, None]) for _ in range(40)]
    zero = [([1, 0, 3], [0, 5], [0.0, 1.5], [2.5, 0.0]) for _ in range(40)]
    check(native, oracle, sch, A.columns_from_rows(sch, zero), data=U.unsafe_rows(sch, rows))
    # garbage bits in the null slots: what the slots hold is encoded
    data, offs = U.unsafe_rows(sch, rows, garbage=True, seed=7)
    enc = native.Encoder(sch)
    try:
        enc.encode_rows(data, offs)
        got = enc.result_host()
    finally:
        enc.close()
    back = []
    for r in range(40):
        row = data[offs[r]:offs[r + 1]].tobytes()
        vals = []
        for f, (t, w) in enumerate([(np.int32, 4), (np.int64, 8), (np.float32, 4), (np.float64, 8)]):
            s = int.from_bytes(row[8 + 8 * f:16 + 8 * f], "little")
            o, n = s >> 32, int.from_bytes(row[(s >> 32):(s >> 32) + 8], "little")
            vals.append(list(np.frombuffer(row[o + 16:o + 16 + n * w], t)))
        back.append(tuple(vals))
    assert any(b != z for b, z in zip(back, zero))
    want, rc, _ = oracle.encode(A.columns_from_rows(sch, back), sch)
    assert rc == 0 and got == want


@pytest.mark.parametrize("case", ["string", "binary", "decimal", "inner_array"])
def test_null_elements_are_npe(native, case):
    rt = TFR_RT_SEQUENCE_EXAMPLE if case == "inner_array" else TFR_RT_EXAMPLE
    dt = {"string": ArrayType(StringType()), "binary": ArrayType(BinaryType()), "decimal": ArrayType(DecimalType()),
          "inner_array": ArrayType(ArrayType(LongType()))}[case]
    good = {"string": ["a", "b"], "binary": [b"x"], "decimal": [1, 2], "inner_array": [[1], []]}[case]
    bad = {"string": ["a", None], "binary": [None], "decimal": [None, 2], "inner_array": [[1], None]}[case]
    sch = StructType([StructField("k", LongType()), StructField("x", dt)])
    rows = [(i, bad if i in (37, 90) else good) for i in range(128)]
    data, offs = U.unsafe_rows(sch, rows)
    code, row = rows_error(native, sch, data, offs, rt)
    assert code == A.TFR_E_NULL_IN_NONNULL and row == 37


def test_null_field_in_nonnullable_is_npe(native):
    sch = StructType([StructField("ok", LongType()), StructField("nn", ArrayType(FloatType()), nullable=False), StructField("z", NullType(), True)])
    data, offs = U.unsafe_rows(sch, [(i, None if i in (41, 77) else [1.0], None) for i in range(100)])
    assert rows_error(native, sch, data, offs) == (A.TFR_E_NULL_IN_NONNULL, 41)


def _malformed_batch():
    sch = StructType([StructField("a", LongType()), StructField("s", StringType()), StructField("v", ArrayType(LongType())),
                      StructField("sa", ArrayType(StringType()))])
    rows = [(i, "s" * (i % 9), list(range(i % 5)), ["x" * (i % 3), "yy"]) for i in range(100)]
    data, offs = U.unsafe_rows(sch, rows)
    return sch, data, offs


def _slot(data, offs, r, f):
    p = int(offs[r]) + 8 + 8 * f
    return p, int.from_bytes(data[p:p + 8].tobytes(), "little")


def _put(data, p, v, n=8):
    data[p:p + n] = np.frombuffer((v & ((1 << (8 * n)) - 1)).to_bytes(n, "little"), np.uint8)


@pytest.mark.parametrize("kind", ["slot_offset", "slot_size", "misaligned_slot", "num_elements_negative", "num_elements_oversized",
                                  "element_offset", "short_row", "misaligned_row", "offsets_decrease"])
def test_malformed_rows_are_invalid_arg(native, kind):
    sch, data, offs = _malformed_batch()
    data, offs = data.copy(), offs.copy()
    k, want = 50, 50
    rlen = int(offs[k + 1] - offs[k])
    if kind == "slot_offset":
        p, s = _slot(data, offs, k, 1); _put(data, p, ((rlen + 8) << 32) | (s & 0xFFFFFFFF))
    elif kind == "slot_size":
        p, s = _slot(data, offs, k, 2); _put(data, p, (s & ~0xFFFFFFFF) | (rlen - (s >> 32) + 1))
    elif kind == "misaligned_slot":
        p, s = _slot(data, offs, k, 2); _put(data, p, s + (4 << 32) - 4)
    elif kind == "num_elements_negative":
        p, s = _slot(data, offs, k, 2); _put(data, int(offs[k]) + (s >> 32), -3)
    elif kind == "num_elements_oversized":
        p, s = _slot(data, offs, k, 2); _put(data, int(offs[k]) + (s >> 32), 1000)
    elif kind == "element_offset":
        p, s = _slot(data, offs, k, 3)
        a = int(offs[k]) + (s >> 32)
        _put(data, a + 16, (4096 << 32) | 2)
    elif kind == "short_row":
        offs[k + 1] = offs[k] + 16                            # shorter than its 40-byte fixed region; row k + 1 starts inside row k
    elif kind == "misaligned_row":
        offs[k] += 4
        want = k - 1                                          # row k - 1 ends on a misaligned offset: it fails first
    elif kind == "offsets_decrease":
        offs[k + 1] = offs[k] - 8
    code, row = rows_error(native, sch, data, offs)
    assert code == A.TFR_E_INVALID_ARG and row == want, (kind, code, row)


def test_malformed_wins_over_null_at_the_same_row(native):
    sch = StructType([StructField("sa", ArrayType(StringType())), StructField("v", ArrayType(LongType()))])
    data, offs = U.unsafe_rows(sch, [(["a", None] if i == 20 else ["a"], [1, 2]) for i in range(64)])
    p, s = _slot(data, offs, 20, 1)
    _put(data, int(offs[20]) + (s >> 32), -1)
    assert rows_error(native, sch, data, offs) == (A.TFR_E_INVALID_ARG, 20)
    data2, offs2 = U.unsafe_rows(sch, [(["a", None] if i == 10 else ["a"], [1, 2]) for i in range(64)])
    p, s = _slot(data2, offs2, 20, 1)
    _put(data2, int(offs2[20]) + (s >> 32), -1)
    assert rows_error(native, sch, data2, offs2) == (A.TFR_E_NULL_IN_NONNULL, 10)


def test_input_variants(native, oracle):
    """host pageable, the pinned row staging, device rows at an address = 8 mod 16"""
    import torch
    from oracle.corpus import mixed_columns
    sch, cols = mixed_columns(2000, seed=8)
    want, rc, _ = oracle.encode(cols, sch)
    data, offs = U.unsafe_rows(sch, rows_of(cols, 2000))
    enc = native.Encoder(sch)
    try:
        enc.encode_rows(data, offs)
        assert enc.result_host() == want
        st = enc.row_staging(len(data))
        st[:len(data)] = data
        enc.encode_rows((st.ctypes.data, len(data), 0), offs)
        assert enc.result_host() == want
        buf = torch.zeros(len(data) + 8, dtype=torch.uint8, device="cuda")
        dev = buf[8:]
        assert dev.data_ptr() % 16 == 8
        dev.copy_(torch.from_numpy(data))
        doffs = torch.from_numpy(offs).cuda()
        ptr, nb = enc.encode_rows(dev, doffs)
        assert enc.result_host() == want
        torch.cuda.synchronize()
    finally:
        enc.close()


def test_one_mib_binary_row_and_reuse_across_sizes(native, oracle):
    """a 1 MiB binary row (its tile is read from global memory), then one encoder across batches of very different row sizes"""
    rng = np.random.default_rng(11)
    sch = StructType([StructField("id", LongType()), StructField("b", BinaryType()), StructField("f", ArrayType(FloatType()))])
    def rows(n, big=None, blen=0):
        out = [(i, rng.integers(0, 256, i % 40, dtype=np.uint8).tobytes(), [float(np.float32(x)) for x in rng.standard_normal(i % 6)]) for i in range(n)]
        if big is not None:
            out[big] = (7, rng.integers(0, 256, blen, dtype=np.uint8).tobytes(), [1.0] * 3000)
        return out
    enc = native.Encoder(sch)
    try:
        for data in (rows(40, big=17, blen=1 << 20), rows(3000), rows(5), rows(900, big=899, blen=300_000), rows(64)):
            cols = A.columns_from_rows(sch, data)
            want, rc, _ = oracle.encode(cols, sch)
            enc.encode_rows(*U.unsafe_rows(sch, data))
            got = enc.result_host()
            assert got == want, _diff(got, want)
    finally:
        enc.close()
    bsch = byte_array_schema()
    big = [(rng.integers(0, 256, s, dtype=np.uint8).tobytes(),) for s in (5, 1 << 20, 0, 77)]
    check(native, oracle, bsch, A.columns_from_rows(bsch, big), TFR_RT_BYTE_ARRAY)
