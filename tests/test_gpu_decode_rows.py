"""GPU tests of tfr_batch_rows: a decoded batch as Spark UnsafeRows.  Every batch is compared byte for byte, offsets
included, with oracle.unsaferow's rows of the oracle's decode of the same bytes (a failure names the first differing row
and field); the device rows go back through tfr_encode_rows to the original framed bytes.
Reference semantics: M/TFRecordDeserializer.scala:21-61 through Spark's UnsafeProjection."""
import numpy as np
import pytest

from oracle import unsaferow as U
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_encode_rows import rows_of
import unsafe_row_reader as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


class _Dev:
    """a device buffer as __cuda_array_interface__ (read through torch)"""
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


def device_rows(batch):
    import torch
    rp, op, n, nb = batch.unsafe_rows(to_host=False)
    offs = torch.as_tensor(_Dev(op, n + 1, "<i8"), device="cuda")
    rows = torch.as_tensor(_Dev(rp, nb, "|u1"), device="cuda") if nb else torch.zeros(0, dtype=torch.uint8, device="cuda")
    return rows, offs, (rp, op, n, nb)


def host_rows(batch):
    rows, offs = batch.unsafe_rows(to_host=True)
    return rows.copy(), offs.copy()


def expected(sch, cols, n):
    data, offs = U.unsafe_rows(sch, rows_of(cols, n))
    return data, offs.astype(np.int64)


def assert_rows(sch, got, want, what=""):
    (gr, go), (wr, wo) = got, want
    ok = np.array_equal(go, wo) and np.array_equal(gr, wr)
    assert ok, f"{what}: {R.first_diff(sch, gr, go, wr, wo)}"


def check_batch(native, oracle, batch, data, sch, rt=0, flags=A.TFR_F_DEFAULT, is_final=True, want_rows=None):
    """host and device rows of `batch` == oracle rows of the oracle's decode of `data`"""
    want = oracle.decode(bytes(data), sch, rt, flags=flags, is_final=is_final)
    n = want.info["n_rows"]
    assert batch.info["n_rows"] == n
    w = want_rows if want_rows is not None else expected(sch, want.columns, n)
    h = host_rows(batch)
    assert_rows(sch, h, w, "host rows")
    dr, do, _ = device_rows(batch)
    assert_rows(sch, (dr.cpu().numpy(), do.cpu().numpy()), w, "device rows")
    return h, (dr.clone(), do.clone())                     # the batch's buffers go away with it


def decode_check(native, oracle, sch, data, rt=0, flags=A.TFR_F_DEFAULT, is_final=True, want_rows=None):
    dec = native.Decoder(sch, rt, 0, flags)
    try:
        b, _ = dec.decode(bytes(data), is_final=is_final)
        out = check_batch(native, oracle, b, data, sch, rt, flags, is_final, want_rows)
        b.release()
        return out
    finally:
        dec.close()


def _has_decimal(sch):
    return any(lower_type(f.dataType)[0] == TFR_T_DECIMAL for f in sch)


def _schema_of_case(c):
    return byte_array_schema() if c.record_type == TFR_RT_BYTE_ARRAY else c.schema


def test_every_case(native, oracle):
    import cases as CS
    n = 0
    for c in CS.all_cases():
        sch = _schema_of_case(c)
        if _has_decimal(sch):
            continue
        flags = getattr(c, "flags", A.TFR_F_DEFAULT)
        decode_check(native, oracle, sch, c.data(), c.record_type, flags=flags, is_final=getattr(c, "is_final", True))
        n += 1
    assert n > 20


def test_golden_vectors(native, oracle):
    import test_golden as G
    import os
    for e in G.INDEX:
        sch = byte_array_schema() if e["record_type"] == 2 else G.schema_of(e)
        if _has_decimal(sch):
            continue
        data = open(os.path.join(G.HERE, e["file"]), "rb").read()
        decode_check(native, oracle, sch, data, e["record_type"], flags=e["flags"], is_final=e["is_final"])


def _roundtrip(native, sch, rt, framed, host, dev):
    """rows -> tfr_encode_rows -> the original framed bytes, from the host rows and from the device rows"""
    import torch
    enc = native.Encoder(sch, rt)
    try:
        enc.encode_rows(host[0], host[1].astype(np.int32))
        assert enc.result_host() == framed
        enc.encode_rows(dev[0], dev[1].to(torch.int32), on_device=True)
        assert enc.result_host() == framed
    finally:
        enc.close()


def test_cfg1(native, oracle):
    from oracle.corpus import cfg1_columns
    sch, cols = cfg1_columns(10_000, seed=41)
    data, rc, _ = oracle.encode(cols, sch)
    h, d = decode_check(native, oracle, sch, data)
    _roundtrip(native, sch, 0, data, h, d)


@pytest.mark.parametrize("n", [1, 31, 5000, 250_000])
def test_cfg2(native, oracle, n):
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(n, seed=7 + n)
    data, rc, _ = oracle.encode(cols, sch)
    wr, wo = U.cfg2_rows(cols)
    h, d = decode_check(native, oracle, sch, data, want_rows=(wr, wo.astype(np.int64)))
    _roundtrip(native, sch, 0, data, h, d)


def test_mixed_columns_with_nulls(native, oracle):
    from oracle.corpus import mixed_columns
    sch, cols = mixed_columns(3000, seed=23)
    data, rc, _ = oracle.encode(cols, sch)
    decode_check(native, oracle, sch, data)


def test_cfg4_sequence_example(native, oracle):
    from oracle.corpus import cfg4_columns
    sch, cols = cfg4_columns(2000, seed=79)
    data, rc, _ = oracle.encode(cols, sch, TFR_RT_SEQUENCE_EXAMPLE)
    h, d = decode_check(native, oracle, sch, data, TFR_RT_SEQUENCE_EXAMPLE)
    _roundtrip(native, sch, TFR_RT_SEQUENCE_EXAMPLE, data, h, d)


def test_bytearray(native, oracle):
    rng = np.random.default_rng(9)
    sch = byte_array_schema()
    rows = [(rng.integers(0, 256, int(s), dtype=np.uint8).tobytes(),) for s in [0, 1, 7, 8, 9, 255, 256, 257, 1024, 5000] + list(rng.integers(0, 1500, 500))]
    cols = A.columns_from_rows(sch, rows, TFR_RT_BYTE_ARRAY)
    data, rc, _ = oracle.encode(cols, sch, TFR_RT_BYTE_ARRAY)
    h, d = decode_check(native, oracle, sch, data, TFR_RT_BYTE_ARRAY)
    _roundtrip(native, sch, TFR_RT_BYTE_ARRAY, data, h, d)


@pytest.mark.parametrize("seed", range(16))
def test_random_schemas(native, oracle, seed):
    from test_gpu_fuzz import _schema, _batch
    rng = np.random.default_rng(500 + seed)
    seq = seed % 2 == 1
    sch, gens = _schema(rng, seq=seq)
    rt = TFR_RT_SEQUENCE_EXAMPLE if seq else TFR_RT_EXAMPLE
    data = _batch(oracle, sch, gens, int(rng.integers(1, 400)), seed, rt)
    decode_check(native, oracle, sch, data, rt)


def test_pipelined_steady_state_and_redo(native, oracle):
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(4000, seed=99)
    data, rc, _ = oracle.encode(cols, sch)
    want = U.cfg2_rows(cols)
    want = (want[0], want[1].astype(np.int64))
    dec = native.Decoder(sch)
    try:
        for it in range(4):                                # first batches learn shapes; then pipelined submits
            b = dec.submit(data)
            if it == 2:
                b.to_host()                                # rows asked for after the Arrow copy ...
            check_batch(native, oracle, b, data, sch, want_rows=want)
            if it == 3:
                b.to_host()                                # ... and before it
                check_batch(native, oracle, b, data, sch, want_rows=want)
            b.release()
        assert dec.stats()["speculative_submits"] >= 1
        # a payload bit flip: the batch is redone, the rows before the failing record only
        bad = bytearray(data)
        bad[len(data) // 2] ^= 0x10
        b = dec.submit(bytes(bad))
        h, _ = check_batch(native, oracle, b, bad, sch)
        assert b.info["error_code"] != 0 and len(h[1]) == b.info["n_rows"] + 1
        b.release()
        b = dec.submit(data)                               # released without ever asking for rows
        b.release()
    finally:
        dec.close()


def test_float_bits(native, oracle):
    sch = StructType([StructField("f", FloatType()), StructField("d", DoubleType()), StructField("af", ArrayType(FloatType())),
                      StructField("ad", ArrayType(DoubleType()))])
    bits = np.array([0x7FC12345, 0xFFC00001, 0x80000000, 0x7F800001, 0x7FA00000, 0, 1, 0xFF800000], np.uint32).view(np.float32)
    rows = [(bits[i], float(bits[i]) if i != 4 else None, list(bits), list(bits[:i])) for i in range(len(bits))]
    cols = A.columns_from_rows(sch, rows)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0
    decode_check(native, oracle, sch, data)


def test_edges(native, oracle):
    sch = StructType([StructField("s", StringType()), StructField("a", ArrayType(LongType())), StructField("as", ArrayType(StringType())),
                      StructField("b", BinaryType())])
    rng = np.random.default_rng(3)
    rows = [("", [], [], b""), ("", [], [""], b""), ("x", [1], ["", "é"], b"\0")]
    rows.append(("y", [2], ["s" * int(k) for k in rng.integers(0, 20, 3000)], rng.integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()))
    rows += [("z" * int(k), list(range(int(k))), ["q"] * int(k % 5), b"w" * int(k)) for k in rng.integers(0, 300, 200)]
    cols = A.columns_from_rows(sch, rows)
    data, rc, _ = oracle.encode(cols, sch)
    decode_check(native, oracle, sch, data)
    # an empty batch
    dec = native.Decoder(sch)
    try:
        b, _ = dec.decode(b"")
        rows_h, offs_h = b.unsafe_rows(True)
        assert len(rows_h) == 0 and list(offs_h) == [0]
        assert b.unsafe_rows(False)[2:] == (0, 0)
        b.release()
    finally:
        dec.close()


def test_calling_rules(native, oracle):
    from oracle.corpus import cfg1_columns
    sch, cols = cfg1_columns(300, seed=5)
    data, rc, _ = oracle.encode(cols, sch)
    dec = native.Decoder(sch)
    try:
        b, _ = dec.decode(data)
        d1 = b.unsafe_rows(False)
        h1 = b.unsafe_rows(True)
        assert b.unsafe_rows(False) == d1                  # the same buffers on a second call
        h2 = b.unsafe_rows(True)
        assert h2[0].ctypes.data == h1[0].ctypes.data and h2[1].ctypes.data == h1[1].ctypes.data
        b.release()
    finally:
        dec.close()
    dsch = StructType([StructField("x", LongType()), StructField("dec", DecimalType())])
    dcols = A.columns_from_rows(dsch, [(1, 1.5)])
    ddata, rc, _ = oracle.encode(dcols, dsch)
    dec = native.Decoder(dsch)
    try:
        b, _ = dec.decode(ddata)
        with pytest.raises(native.TfrError) as ei:
            b.unsafe_rows(True)
        assert ei.value.code == A.TFR_E_UNSUPPORTED_TYPE and "dec" in str(ei.value)
        assert b.to_host()[0].n_rows == 1                  # the columns stay usable
        b.release()
    finally:
        dec.close()
