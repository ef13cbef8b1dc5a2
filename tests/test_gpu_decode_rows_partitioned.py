"""GPU tests of tfr_batch_rows_with_partition: a decoded batch as Spark UnsafeRows of D ++ P, the file's partition values
appended to every row.  Host and device rows, int64 offsets included, are compared byte for byte with
partition_rows' joined rows of the oracle's decode (written from values); a failure names the first differing row and
field.  Semantics: include/tfrgpu.h, DESIGN.md section 2."""
import struct

import numpy as np
import pytest

import partition_rows as P
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_decode_rows import _Dev, _has_decimal, _schema_of_case, native  # noqa: F401 (fixture)
from test_gpu_encode_rows import rows_of

pytestmark = pytest.mark.gpu

FIXED_PART = (["string", "int", ("decimal", 38, 6)], ["2024-05-01", 17, None])


def _names(sch, pt):
    return [f.name for f in sch] + [f"partition[{j}] {t}" for j, t in enumerate(pt)]


def first_diff(sch, pt, got, want) -> str:
    (gr, go), (wr, wo) = got, want
    if len(go) != len(wo):
        return f"{len(go) - 1} rows vs {len(wo) - 1}"
    names = _names(sch, pt)
    nf = len(names)
    nw = (nf + 63) // 64
    for r in range(len(wo) - 1):
        g, w = bytes(gr[go[r]:go[r + 1]]), bytes(wr[wo[r]:wo[r + 1]])
        if go[r] == wo[r] and g == w:
            continue
        if go[r] != wo[r] or len(g) != len(w):
            return f"row {r}: offset {go[r]} size {len(g)} vs offset {wo[r]} size {len(w)}"
        at = next(i for i in range(len(w)) if g[i] != w[i])
        if at < 8 * nw:
            bit = 8 * at + next(b for b in range(8) if (g[at] ^ w[at]) >> b & 1)
            return f"row {r}: null bit {bit} ({names[bit] if bit < nf else 'beyond the fields'})"
        if at < 8 * (nw + nf):
            return f"row {r}: slot of {names[(at - 8 * nw) // 8]}"
        owner = max(((struct.unpack_from('<Q', w, 8 * (nw + i))[0] >> 32, names[i]) for i in range(nf)
                     if struct.unpack_from('<Q', w, 8 * (nw + i))[0] >> 32 <= at), default=(0, "?"))
        return f"row {r}: variable byte {at}, in the value of {owner[1]}"
    return "no difference"


def assert_rows(sch, pt, got, want, what):
    ok = np.array_equal(got[1], want[1]) and np.array_equal(got[0], want[0])
    assert ok, f"{what}: {first_diff(sch, pt, got, want)}"


def device_rows(batch, part):
    import torch
    rp, op, n, nb = batch.unsafe_rows(False, part)
    offs = torch.as_tensor(_Dev(op, n + 1, "<i8"), device="cuda")
    rows = torch.as_tensor(_Dev(rp, nb, "|u1"), device="cuda") if nb else torch.zeros(0, dtype=torch.uint8, device="cuda")
    return rows, offs


def check_batch(oracle, batch, data, sch, pt, pv, rt=0, flags=A.TFR_F_DEFAULT, is_final=True, want=None):
    """host and device rows of `batch` with partition values pv == the joined rows of the oracle's decode of `data`"""
    if want is None:
        wd = oracle.decode(bytes(data), sch, rt, flags=flags, is_final=is_final)
        want = P.joined_rows(sch, rows_of(wd.columns, wd.info["n_rows"]), pt, pv)
    assert batch.info["n_rows"] == len(want[1]) - 1
    part = (P.partition_row(pt, pv), P.var_flags(pt))
    hr, ho = batch.unsafe_rows(True, part)
    h = (hr.copy(), ho.copy())
    assert_rows(sch, pt, h, want, "host rows")
    dr, do = device_rows(batch, part)
    d = (dr.cpu().numpy(), do.cpu().numpy())
    assert_rows(sch, pt, d, want, "device rows")
    return h, (dr.clone(), do.clone())


def decode_check(native, oracle, sch, data, pt, pv, rt=0, flags=A.TFR_F_DEFAULT, is_final=True, want=None):
    dec = native.Decoder(sch, rt, 0, flags)
    try:
        b, _ = dec.decode(bytes(data), is_final=is_final)
        out = check_batch(oracle, b, data, sch, pt, pv, rt, flags, is_final, want)
        b.release()
        return out
    finally:
        dec.close()


def _small_mixed(n=300, seed=1):
    sch = StructType([StructField("i", IntegerType()), StructField("s", StringType()), StructField("al", ArrayType(LongType())),
                      StructField("d", DoubleType())])
    rng = np.random.default_rng(seed)
    rows = [(int(rng.integers(-9, 9)) if k % 7 else None, "v" * int(k % 11) if k % 5 else None,
             list(range(int(k % 4))) if k % 3 else None, float(k) / 3) for k in range(n)]
    return sch, A.columns_from_rows(sch, rows)


def _value(t, rng):
    if isinstance(t, tuple):                                    # the unscaled value
        if t[1] > 18:
            return int(rng.integers(-10 ** 18, 10 ** 18)) * 10 ** (t[1] - 19) + int(rng.integers(0, 10))
        return int(rng.integers(-(10 ** t[1] - 1), 10 ** t[1]))
    return {"boolean": bool(rng.integers(0, 2)), "byte": int(rng.integers(-128, 128)), "short": int(rng.integers(-2 ** 15, 2 ** 15)),
            "int": int(rng.integers(-2 ** 31, 2 ** 31)), "date": int(rng.integers(-10 ** 5, 10 ** 5)),
            "long": int(rng.integers(-2 ** 63, 2 ** 63)), "timestamp": int(rng.integers(-2 ** 62, 2 ** 62)),
            "float": float(np.float32(rng.normal())), "double": float(rng.normal()),
            "string": "p" * int(rng.integers(0, 20)), "binary": rng.integers(0, 256, int(rng.integers(0, 30)), dtype=np.uint8).tobytes()}[t]


def _random_partition(rng, n_fields, null_rate=0.3):
    pt = [P.PART_TYPES[int(i)] for i in rng.integers(0, len(P.PART_TYPES), n_fields)]
    pv = [None if rng.random() < null_rate else _value(t, rng) for t in pt]
    return pt, pv


# 1. each partition type, non-null and null, behind a small mixed data schema; and all of them at once
@pytest.mark.parametrize("t", P.PART_TYPES, ids=str)
def test_each_partition_type(native, oracle, t):
    sch, cols = _small_mixed()
    data, rc, _ = oracle.encode(cols, sch)
    rng = np.random.default_rng(5)
    for v in [_value(t, rng), None]:
        decode_check(native, oracle, sch, data, [t], [v])


def test_every_type_at_once(native, oracle):
    sch, cols = _small_mixed(500, 2)
    data, rc, _ = oracle.encode(cols, sch)
    rng = np.random.default_rng(6)
    pt = list(P.PART_TYPES)
    decode_check(native, oracle, sch, data, pt, [_value(t, rng) for t in pt])
    decode_check(native, oracle, sch, data, pt, [None] * len(pt))
    decode_check(native, oracle, sch, data, pt + pt, [_value(t, rng) for t in pt] + [None] * len(pt))


# 2. null-bitset boundaries
@pytest.mark.parametrize("nd,np_", [(63, 1), (64, 1), (60, 8), (0, 1), (0, 65), (1, 127)])
def test_bitset_boundaries(native, oracle, nd, np_):
    rng = np.random.default_rng(nd * 1000 + np_)
    pt, pv = _random_partition(rng, np_)
    if nd == 0:                                                 # no data fields: the records' features are all skipped
        data = _z_records(oracle, 70)
        prow = P.partition_row(pt, pv)
        want = (np.frombuffer(prow * 70, np.uint8), np.arange(71, dtype=np.int64) * len(prow))
        decode_check(native, oracle, StructType([]), data, pt, pv, want=want)
        return
    sch = StructType([StructField(f"c{i}", [LongType(), StringType(), FloatType()][i % 3]) for i in range(nd)])
    rows = [tuple(None if rng.random() < 0.2 else [int(k + i), "s" * (i % 9), float(i)][i % 3] for i in range(nd)) for k in range(70)]
    cols = A.columns_from_rows(sch, rows)
    data, rc, _ = oracle.encode(cols, sch)
    decode_check(native, oracle, sch, data, pt, pv)


def _z_records(oracle, n):
    z = StructType([StructField("z", LongType())])
    data, rc, _ = oracle.encode(A.columns_from_rows(z, [(k,) for k in range(n)]), z)
    return data


@pytest.mark.parametrize("n", [1, 31, 5000, 250_000])
def test_cfg2_with_string_and_int(native, oracle, n):
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(n, seed=7 + n)
    data, rc, _ = oracle.encode(cols, sch)
    pt, pv = ["string", "int"], ["2024-05-01", 20240501]
    want = P.cfg2_joined_rows(cols, pt, pv)
    m = min(n, 40)                                              # the vectorised rows against the value writer on a prefix
    wr, wo = P.joined_rows(sch, rows_of(cols, m), pt, pv)
    assert np.array_equal(want[0][:wo[-1]], wr) and np.array_equal(want[1][:m + 1], wo)
    decode_check(native, oracle, sch, data, pt, pv, want=want)


# 3. every case and golden vector with one fixed partition row: the rows stop at the first bad record
def test_every_case(native, oracle):
    import cases as CS
    n = 0
    for c in CS.all_cases():
        sch = _schema_of_case(c)
        if _has_decimal(sch):
            continue
        decode_check(native, oracle, sch, c.data(), *FIXED_PART, c.record_type, flags=getattr(c, "flags", A.TFR_F_DEFAULT),
                     is_final=getattr(c, "is_final", True))
        n += 1
    assert n > 20


def test_golden_vectors(native, oracle):
    import os
    import test_golden as G
    for e in G.INDEX:
        sch = byte_array_schema() if e["record_type"] == 2 else G.schema_of(e)
        if _has_decimal(sch):
            continue
        data = open(os.path.join(G.HERE, e["file"]), "rb").read()
        decode_check(native, oracle, sch, data, *FIXED_PART, e["record_type"], flags=e["flags"], is_final=e["is_final"])


# 4. SequenceExamples, ByteArray, random data schemas with random partition schemas
def test_sequence_example(native, oracle):
    from oracle.corpus import cfg4_columns
    sch, cols = cfg4_columns(2000, seed=79)
    data, rc, _ = oracle.encode(cols, sch, TFR_RT_SEQUENCE_EXAMPLE)
    decode_check(native, oracle, sch, data, *FIXED_PART, TFR_RT_SEQUENCE_EXAMPLE)


def test_bytearray(native, oracle):
    rng = np.random.default_rng(9)
    sch = byte_array_schema()
    rows = [(rng.integers(0, 256, int(s), dtype=np.uint8).tobytes(),) for s in [0, 1, 7, 8, 255, 256, 257, 5000] + list(rng.integers(0, 1500, 300))]
    cols = A.columns_from_rows(sch, rows, TFR_RT_BYTE_ARRAY)
    data, rc, _ = oracle.encode(cols, sch, TFR_RT_BYTE_ARRAY)
    decode_check(native, oracle, sch, data, *_random_partition(rng, 9), TFR_RT_BYTE_ARRAY)


@pytest.mark.parametrize("seed", range(16))
def test_random_schemas(native, oracle, seed):
    from test_gpu_fuzz import _schema, _batch
    rng = np.random.default_rng(500 + seed)
    seq = seed % 2 == 1
    sch, gens = _schema(rng, seq=seq)
    rt = TFR_RT_SEQUENCE_EXAMPLE if seq else TFR_RT_EXAMPLE
    data = _batch(oracle, sch, gens, int(rng.integers(1, 400)), seed, rt)
    prng = np.random.default_rng(900 + seed)
    decode_check(native, oracle, sch, data, *_random_partition(prng, int(prng.integers(1, 71)), prng.random()), rt)


# 5. pipelined, redone and released-unasked batches
def test_pipelined_steady_state_and_redo(native, oracle):
    from oracle.corpus import cfg2_columns
    sch, cols = cfg2_columns(4000, seed=99)
    data, rc, _ = oracle.encode(cols, sch)
    pt, pv = FIXED_PART
    want = P.cfg2_joined_rows(cols, pt, pv)
    dec = native.Decoder(sch)
    try:
        for it in range(4):
            b = dec.submit(data)
            if it == 2:
                b.to_host()
            check_batch(oracle, b, data, sch, pt, pv, want=want)
            b.release()
        assert dec.stats()["speculative_submits"] >= 1
        bad = bytearray(data)
        bad[len(data) // 2] ^= 0x10
        b = dec.submit(bytes(bad))
        h, _ = check_batch(oracle, b, bad, sch, pt, pv)
        assert b.info["error_code"] != 0 and len(h[1]) == b.info["n_rows"] + 1
        b.release()
        b = dec.submit(data)
        b.release()
    finally:
        dec.close()


# 6. a 1 MiB partition value, an empty string, an empty batch, an empty data schema
def test_one_mib_partition_value(native, oracle):
    import torch
    sch = StructType([StructField("x", LongType())])
    n = 10_000
    cols = A.columns_from_rows(sch, [(k * 7,) for k in range(n)])
    data, rc, _ = oracle.encode(cols, sch)
    big = np.random.default_rng(1).integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()
    pt, pv = ["binary", "int"], [big, 3]
    # every row has the same size: the value writer on the first rows, then the rest checked as one 2-D view
    head = P.joined_rows(sch, [(k * 7,) for k in range(4)], pt, pv)
    size = int(head[1][1])
    assert size == 8 * (1 + 3) + (1 << 20)
    want_first = np.frombuffer(P.joined_row(sch, (0,), pt, pv), np.uint8)
    part = (P.partition_row(pt, pv), P.var_flags(pt))
    dec = native.Decoder(sch)
    try:
        b, _ = dec.decode(data)
        dr, do = device_rows(b, part)
        assert torch.equal(do.cpu(), torch.arange(n + 1, dtype=torch.int64) * size)
        D = dr.view(n, size)
        ref = torch.as_tensor(want_first.copy(), device="cuda")
        got4 = D[:4].reshape(-1).cpu().numpy()
        assert np.array_equal(got4, head[0]), first_diff(sch, pt, (got4, head[1]), head)
        # the rest: null word zero, the data slot k * 7, everything from the partition slots on equal to row 0's
        assert not D[:, :8].any().item()
        assert torch.equal(D[:, 8:16].contiguous().view(torch.int64).view(-1).cpu(), torch.arange(n, dtype=torch.int64) * 7)
        for r0 in range(0, n, 1000):
            assert torch.equal(D[r0:r0 + 1000, 16:], ref[16:].expand(min(1000, n - r0), size - 16)), f"device rows {r0}.."
        hr, ho = b.unsafe_rows(True, part)
        assert np.array_equal(ho, np.arange(n + 1, dtype=np.int64) * size)
        H = hr.reshape(n, size)
        assert not H[:, :8].any()
        assert np.array_equal(H[:, 8:16].copy().view(np.int64).reshape(-1), np.arange(n, dtype=np.int64) * 7)
        for r0 in range(0, n, 1000):
            assert (H[r0:r0 + 1000, 16:] == want_first[16:]).all(), f"host rows {r0}.."
        b.release()
    finally:
        dec.close()


def test_empty_string_empty_batch_empty_schema(native, oracle):
    sch, cols = _small_mixed(100, 3)
    data, rc, _ = oracle.encode(cols, sch)
    decode_check(native, oracle, sch, data, ["string", "binary"], ["", b""])
    pt, pv = FIXED_PART
    part = (P.partition_row(pt, pv), P.var_flags(pt))
    dec = native.Decoder(sch)
    try:
        b, _ = dec.decode(b"")
        rows_h, offs_h = b.unsafe_rows(True, part)
        assert len(rows_h) == 0 and list(offs_h) == [0]
        assert b.unsafe_rows(False, part)[2:] == (0, 0)
        b.release()
    finally:
        dec.close()
    # no data fields: every row is the partition row itself
    empty = StructType([])
    n = 37
    edata = _z_records(oracle, n)
    for pt, pv in [FIXED_PART, (["int"], [None]), _random_partition(np.random.default_rng(4), 65)]:
        prow = P.partition_row(pt, pv)
        want = (np.frombuffer(prow * n, np.uint8), np.arange(n + 1, dtype=np.int64) * len(prow))
        decode_check(native, oracle, empty, edata, pt, pv, want=want)


# 7. calling rules
def _raw(native, b, to_host, row, nbytes, np_, flags):
    import ctypes as C
    rp, op, n, nb = C.c_void_p(), C.c_void_p(), C.c_int64(), C.c_size_t()
    return native.lib().tfr_batch_rows_with_partition(b.h, to_host, row, nbytes, np_, flags, C.byref(rp), C.byref(op), C.byref(n), C.byref(nb))


def test_calling_rules(native, oracle):
    from oracle.corpus import cfg1_columns
    sch, cols = cfg1_columns(300, seed=5)
    data, rc, _ = oracle.encode(cols, sch)
    pt, pv = FIXED_PART
    part = (P.partition_row(pt, pv), P.var_flags(pt))
    dec = native.Decoder(sch)
    try:
        # np = 0 is tfr_batch_rows
        b1, _ = dec.decode(data)
        b2, _ = dec.decode(data)
        r1 = b1.unsafe_rows(True)
        r2 = b2.unsafe_rows(True, (b"", b""))
        assert np.array_equal(r1[0], r2[0]) and np.array_equal(r1[1], r2[1])
        assert b1.unsafe_rows(True, (b"", b""))[0].ctypes.data == r1[0].ctypes.data      # the same rows: np = 0 both
        b1.release()
        b2.release()
        # the same partition row again: the same buffers; another one, or none: INVALID_ARG, the batch stays usable
        b, _ = dec.decode(data)
        d1 = b.unsafe_rows(False, part)
        h1 = b.unsafe_rows(True, part)
        assert b.unsafe_rows(False, (bytearray(part[0]), list(part[1]))) == d1
        h2 = b.unsafe_rows(True, part)
        assert h2[0].ctypes.data == h1[0].ctypes.data and h2[1].ctypes.data == h1[1].ctypes.data
        other = [(P.partition_row(pt, ["2024-05-02", 17, None]), part[1]), (part[0], bytes([1, 1, 1])), None,
                 (P.partition_row(pt + ["int"], pv + [1]), P.var_flags(pt + ["int"]))]
        for o in other:
            with pytest.raises(native.TfrError) as ei:
                b.unsafe_rows(True, o)
            assert ei.value.code == A.TFR_E_INVALID_ARG
        assert b.to_host()[0].n_rows == 300
        h3 = b.unsafe_rows(True, part)
        assert np.array_equal(h3[1], h1[1]) and np.array_equal(h3[0][:h1[1][2]], h1[0][:h1[1][2]])
        # malformed partition rows, each checked before any work
        one = P.partition_row(["string"], ["abc"])                 # 8 null + 8 slot + 8 value bytes
        slot = lambda off, size: one[:8] + struct.pack("<Q", (off << 32) | size) + one[16:]
        bad = [
            (one, len(one), -1, b"\1", "outside"), (one, len(one), 4097, b"\1" * 4097, "outside"),
            (None, 24, 1, b"\1", "null"), (one, len(one), 1, None, "null"),
            (one, 20, 1, b"\1", "multiple of 8"), (one[:8], 8, 1, b"\1", "fixed region"), (one, 24, 0, b"", "without fields"),
            (b"\2" + one[1:], 24, 1, b"\1", "partition field 1"), (b"\0" * 7 + b"\x80" + one[8:], 24, 1, b"\1", "partition field 63"),
            (slot(12, 3), 24, 1, b"\1", "partition field 0"), (slot(8, 3), 24, 1, b"\1", "partition field 0"),
            (slot(16, 9), 24, 1, b"\1", "partition field 0"), (slot(256, 0), 24, 1, b"\1", "partition field 0"),
        ]
        b2, _ = dec.decode(data)
        for row, nbytes, np_, flags, msg in bad:
            rc = _raw(native, b2, 1, row, nbytes, np_, flags)
            assert rc == A.TFR_E_INVALID_ARG, msg
            assert msg in native.lib().tfr_last_error().decode(), (msg, native.lib().tfr_last_error())
        assert _raw(native, b2, 1, slot(16, 8), 24, 1, b"\1") == 0      # the edge cases are valid: offset 16 .. 24
        assert _raw(native, b2, 1, slot(12, 3), 24, 1, b"\0") != 0      # same row, other flags: not the rows built
        b2.release()
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
            b.unsafe_rows(True, part)
        assert ei.value.code == A.TFR_E_UNSUPPORTED_TYPE and "dec" in str(ei.value)
        assert b.to_host()[0].n_rows == 1
        b.release()
    finally:
        dec.close()


# 8. round trip: rows with encoder-typed partition columns through tfr_encode_rows == the data plus constant columns
def test_roundtrip_through_encode_rows(native, oracle):
    import torch
    sch, cols = _small_mixed(400, 8)
    data, rc, _ = oracle.encode(cols, sch)
    pt = ["int", "long", "float", "double", "string", "binary"]
    pv = [-5, 1 << 40, 1.5, -2.25, "part", b"\x00\xff"]
    ptypes = [IntegerType(), LongType(), FloatType(), DoubleType(), StringType(), BinaryType()]
    full = StructType(list(sch) + [StructField(f"p{j}", t) for j, t in enumerate(ptypes)])
    n = 400
    fcols = A.columns_from_rows(full, [r + tuple(pv) for r in rows_of(cols, n)])
    framed, rc, _ = oracle.encode(fcols, full)
    h, d = decode_check(native, oracle, sch, data, pt, pv)
    enc = native.Encoder(full)
    try:
        enc.encode_rows(h[0], h[1].astype(np.int32))
        assert enc.result_host() == framed
        enc.encode_rows(d[0], d[1].to(torch.int32), on_device=True)
        assert enc.result_host() == framed
    finally:
        enc.close()
