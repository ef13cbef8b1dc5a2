"""GPU parity tests proper: the CUDA decode path through the C ABI vs the CPU oracle, bit-exact.
Run on an H100:  python -m pytest tests -m gpu"""
import numpy as np
import pytest

import cases as CS
from util import assert_columns_equal
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

pytestmark = pytest.mark.gpu
ALL = CS.all_cases()


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def gpu_decode(native, data, schema, record_type=0, flags=A.TFR_F_DEFAULT, is_final=True):
    dec = native.Decoder(schema, record_type, 0, flags)
    try:
        batch, used = dec.decode(data, is_final=is_final)
        cols = batch.to_host()
        info = dict(batch.info)
        batch.release()
        return cols, info, used
    finally:
        dec.close()


@pytest.mark.parametrize("case", ALL, ids=[c.name for c in ALL])
def test_case_matches_oracle(native, oracle, case):
    data = case.data()
    want = oracle.decode(data, case.schema, case.record_type, flags=case.flags, is_final=case.is_final)
    got, info, used = gpu_decode(native, data, case.schema, case.record_type, case.flags, case.is_final)
    wi = want.info
    assert info["error_code"] == wi["error_code"], (A.STATUS_NAMES.get(info["error_code"]), A.STATUS_NAMES.get(wi["error_code"]))
    assert info["error_row"] == wi["error_row"]
    assert info["error_field"] == wi["error_field"]
    assert info["n_rows"] == wi["n_rows"]
    assert used == wi["consumed_bytes"]
    names = ["byteArray"] if case.record_type == 2 else case.schema.names
    assert_columns_equal(got, want.columns, names, case.name)
    if case.error is not None:
        assert info["error_code"] == case.error


def _roundtrip(native, oracle, schema, cols, record_type=0, tag=""):
    data, rc, _ = oracle.encode(cols, schema, record_type)
    assert rc == 0
    want = oracle.decode(data, schema, record_type)
    got, info, used = gpu_decode(native, data, schema, record_type)
    assert info["error_code"] == 0, info
    assert used == len(data)
    assert_columns_equal(got, want.columns, schema.names, tag + " vs oracle")
    assert_columns_equal(got, cols, schema.names, tag + " vs source")
    return data


def test_cfg1_10k_rows(native, oracle):
    from oracle.corpus import cfg1_columns
    sch, cols = cfg1_columns(10_000, seed=1234)
    _roundtrip(native, oracle, sch, cols, tag="cfg1")


@pytest.mark.parametrize("n,small", [(1, False), (33, False), (5000, False), (5000, True)])
def test_cfg2_records(native, oracle, n, small):
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(n, seed=2024 + n, small_ints=small)
    _roundtrip(native, oracle, sch, cols, tag=f"cfg2[{n}]")


def test_mixed_types_with_nulls(native, oracle):
    from oracle.corpus import mixed_columns
    sch, cols = mixed_columns(4000, seed=5)
    _roundtrip(native, oracle, sch, cols, tag="mixed")


def test_cfg4_sequence_example(native, oracle):
    from oracle.corpus import cfg4_columns
    sch, cols = cfg4_columns(1500, seed=77, mean_steps=64)
    _roundtrip(native, oracle, sch, cols, record_type=TFR_RT_SEQUENCE_EXAMPLE, tag="cfg4")


def test_column_pruning_and_reorder(native, oracle):
    """requiredSchema reaches the parser (M/DefaultSource.scala:134): a subset in another order"""
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(3000, seed=9)
    data, rc, _ = oracle.encode(cols, sch)
    pick = [40, 3, 63, 17, 0]
    sub = StructType([sch[i] for i in pick] + [StructField("not_there", ArrayType(StringType()))])
    want = oracle.decode(data, sub)
    got, info, _ = gpu_decode(native, data, sub)
    assert info["error_code"] == 0
    assert_columns_equal(got, want.columns, sub.names, "pruned")
    assert_columns_equal(got[:5], [cols[i] for i in pick], sub.names[:5], "pruned vs source")
    assert got[5].null_count == 3000


def test_bytearray_records(native, oracle):
    rng = np.random.default_rng(3)
    sizes = [0, 1, 3, 4, 5, 31, 32, 33, 127, 128, 129, 4095, 4096, 70000] + list(rng.integers(0, 3000, 500))
    rows = [(rng.integers(0, 256, int(s), dtype=np.uint8).tobytes(),) for s in sizes]
    sch = byte_array_schema()
    cols = A.columns_from_rows(sch, rows)
    _roundtrip(native, oracle, sch, cols, record_type=TFR_RT_BYTE_ARRAY, tag="bytearray")


def test_crc_every_alignment_and_length(native, oracle):
    """payload CRC over every (start alignment, length) combination around the 128-byte row size"""
    from oracle import pyref
    rng = np.random.default_rng(11)
    payloads = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in list(range(0, 300)) + [1023, 1024, 1025, 5000]]
    data = b"".join(pyref.frame_fast(p) for p in payloads)
    want = oracle.decode(data, byte_array_schema(), 2)
    got, info, _ = gpu_decode(native, data, byte_array_schema(), 2)
    assert info["error_code"] == 0 and info["n_rows"] == len(payloads)
    assert_columns_equal(got, want.columns, ["byteArray"], "crc sweep")
    # flip one bit in each payload in turn -> CRC_DATA at exactly that record
    for i in [1, 2, 5, 64, 129, 200, len(payloads) - 1]:
        pos = sum(16 + len(p) for p in payloads[:i]) + 12 + len(payloads[i]) // 2
        bad = bytearray(data); bad[pos] ^= 1
        _, info, _ = gpu_decode(native, bytes(bad), byte_array_schema(), 2)
        assert info["error_code"] == A.TFR_E_CRC_DATA and info["error_row"] == i and info["n_rows"] == i


def test_streaming_blocks_carry_partial_records(native, oracle):
    """buildReader stages a file in blocks: non-final blocks leave the partial tail unconsumed"""
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(2000, seed=4)
    data, rc, _ = oracle.encode(cols, sch)
    dec = native.Decoder(sch)
    pos, rows, block = 0, 0, 300_000
    parts = []
    while pos < len(data):
        end = min(len(data), pos + block)
        batch, used = dec.decode(data[pos:end], is_final=end == len(data))
        assert batch.info["error_code"] == 0
        parts.append(batch.to_host())
        rows += batch.n_rows
        batch.release()
        assert used > 0
        pos += used
    dec.close()
    assert rows == 2000
    i64 = np.concatenate([p[0].values for p in parts])
    assert np.array_equal(i64, cols[0].values)
    f = np.concatenate([p[32].values for p in parts])
    assert np.array_equal(f.view(np.uint32), cols[32].values.view(np.uint32))


def test_device_resident_input_and_arrow_export(native, oracle):
    import torch
    import pyarrow as pa
    from oracle.corpus import mixed_columns
    sch, cols = mixed_columns(1000, seed=8)
    data, rc, _ = oracle.encode(cols, sch)
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    dec = native.Decoder(sch)
    batch, used = dec.decode(t)
    assert used == len(data) and batch.info["error_code"] == 0
    arrs = batch.to_arrow()
    want = oracle.decode(data, sch)
    for name, arr, col in zip(sch.names, arrs, want.columns):
        arr.validate(full=True)
        assert len(arr) == 1000 and arr.null_count == col.null_count, name
        py = arr.to_pylist()
        for r in range(0, 1000, 37):
            w = col.get(r)
            g = py[r]
            if isinstance(w, float) or (isinstance(w, list) and w and isinstance(w[0], float)):
                assert np.array_equal(np.array(g, dtype=np.float64), np.array(w, dtype=np.float64), equal_nan=True), name
            else:
                assert g == w, (name, r)
    batch.release()
    dec.close()


def test_frame_speculation_repair_paths(native, oracle):
    """records much larger than a chunk + payloads that embed valid TFRecord streams"""
    from oracle import pyref
    rng = np.random.default_rng(2)
    inner = b"".join(pyref.frame_fast(rng.integers(0, 256, 50, dtype=np.uint8).tobytes()) for _ in range(3000))
    pay = [inner, b"x" * 5, inner[:100_000], rng.integers(0, 256, 300_000, dtype=np.uint8).tobytes(), b"", inner]
    pay += [rng.integers(0, 256, int(s), dtype=np.uint8).tobytes() for s in rng.integers(0, 9000, 400)]
    data = b"".join(pyref.frame_fast(p) for p in pay)
    want = oracle.decode(data, byte_array_schema(), 2)
    got, info, used = gpu_decode(native, data, byte_array_schema(), 2)
    assert info["error_code"] == 0 and info["n_rows"] == len(pay) and used == len(data)
    assert info["frame_repairs"] > 0
    assert_columns_equal(got, want.columns, ["byteArray"], "repair")


def test_fast_path_learns_then_speculates_then_recovers(native, oracle):
    """tile fast path: batch 1 runs in count mode and learns the shapes, batch 2+ write uniform columns in the
    same pass (speculation), a batch with a different shape falls back to the general path -- all bit-exact"""
    from oracle.corpus import cfg2_columns
    dec = native.Decoder(cfg2_columns(1, seed=1)[0])
    try:
        for i, (n, fl) in enumerate([(3000, 8), (3100, 8), (2900, 8), (2000, 5), (2500, 8)]):
            sch, cols = cfg2_columns(n, seed=100 + i, float_len=fl)
            data, rc, _ = oracle.encode(cols, sch)
            batch, used = dec.decode(data)
            assert batch.info["error_code"] == 0 and used == len(data)
            assert_columns_equal(batch.to_host(), cols, sch.names, f"speculation batch {i}")
            batch.release()
        # ragged lengths inside one batch + nulls: never uniform
        from oracle.corpus import mixed_columns
    finally:
        dec.close()
    sch, cols = cfg2_columns(4000, seed=5)
    # a corrupt record in the middle of a speculating decoder: error semantics must still be exact
    data, rc, _ = oracle.encode(cols, sch)
    dec = native.Decoder(sch)
    try:
        for _ in range(2):
            b, _ = dec.decode(data); b.release()
        bad = bytearray(data); bad[len(data) // 3] ^= 0x20
        want = oracle.decode(bytes(bad), sch)
        b, used = dec.decode(bytes(bad))
        assert b.info["error_code"] == want.info["error_code"] != 0
        assert b.info["error_row"] == want.info["error_row"] and used == want.info["consumed_bytes"]
        assert_columns_equal(b.to_host(), want.columns, sch.names, "error under speculation")
        b.release()
        b, used = dec.decode(data)
        assert b.info["error_code"] == 0
        assert_columns_equal(b.to_host(), cols, sch.names, "after error")
        b.release()
    finally:
        dec.close()


@pytest.mark.parametrize("env", [{"TFR_DISABLE_FAST": "1"}, {}])
def test_path_variants_agree(native, oracle, env, monkeypatch):
    """general path only / other tile geometries: same bits"""
    from oracle.corpus import cfg2_columns, mixed_columns
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for sch, cols in (cfg2_columns(6000, seed=77), mixed_columns(3000, seed=78)):
        data, rc, _ = oracle.encode(cols, sch)
        dec = native.Decoder(sch)
        for _ in range(3):
            b, used = dec.decode(data)
            assert b.info["error_code"] == 0 and used == len(data)
            assert_columns_equal(b.to_host(), cols, sch.names, str(env))
            b.release()
        dec.close()


def test_device_input_at_every_alignment(native, oracle):
    """a device buffer at any byte alignment is legal input (only 16-byte aligned ones take the tile kernels)"""
    import torch
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(700, seed=41)
    data, rc, _ = oracle.encode(cols, sch)
    want = oracle.decode(data, sch)
    dec = native.Decoder(sch)
    try:
        for shift in (0, 1, 3, 4, 8, 15, 16):
            buf = torch.zeros(len(data) + 64, dtype=torch.uint8, device="cuda")
            view = buf[shift:shift + len(data)]
            view.copy_(torch.frombuffer(bytearray(data), dtype=torch.uint8))
            for _ in range(2):                                   # second call: uniform-shape speculation
                batch, used = dec.decode(view)
                assert used == len(data) and batch.info["error_code"] == 0
                assert_columns_equal(batch.to_host(), want.columns, sch.names, f"shift {shift}")
                batch.release()
    finally:
        dec.close()


def test_tile_slot_shapes(native, oracle):
    """record sizes around the tile kernel's slot geometry: tiny payloads (no 16-byte chunk), payloads that end on every
    residue mod 16, one long record among short ones (slot stride follows the longest), Int64 varints of every width"""
    rng = np.random.default_rng(77)
    sch = StructType([StructField("a", LongType()), StructField("s", BinaryType()), StructField("v", ArrayType(LongType()))])
    rows = []
    for i in range(400):
        width = i % 11                                           # 0: small value; k: a value that needs k varint bytes
        a = int(rng.integers(0, 100)) if width == 0 else (-(i + 1) if width == 10 else int(1 << (7 * width - 1)) + i)
        s = rng.integers(0, 256, i % 53, dtype=np.uint8).tobytes()
        v = [int(x) for x in rng.integers(-2**62, 2**62, i % 5)]
        rows.append((a, s, v))
    rows.append((7, rng.integers(0, 256, 5000, dtype=np.uint8).tobytes(), list(range(300))))      # one long record
    rows += [(1, b"", []), (2, b"x", [0])] * 20
    cols = A.columns_from_rows(sch, rows)
    _roundtrip(native, oracle, sch, cols, tag="slot shapes")
    # a single field: payloads of a few bytes only
    sch1 = StructType([StructField("a", LongType())])
    _roundtrip(native, oracle, sch1, A.columns_from_rows(sch1, [(i,) for i in range(100)]), tag="tiny payloads")
