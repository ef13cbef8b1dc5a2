"""GPU tests of the large-record kernels (csrc/large.cuh): Example and ByteArray batches whose records are too large for a
shared-memory tile decode on the pipelined, single-pass path.  Every result is compared with the C oracle's decode of the same
bytes (columns byte for byte, host copy, UnsafeRows); malformed data with the oracle-derived expectation of the drop-mode
suite.  The contract is asserted from Decoder.stats(): after the learning batch every submit is speculative, nothing is
redone or goes through the general kernels, and large_record_batches counts the batches."""
import random

import numpy as np
import pytest

from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa
from test_gpu_decode_rows import check_batch
import partition_rows as P
import test_gpu_decode_rows_pipelined as RP
import test_gpu_drop_malformed as D
import test_gpu_permissive as PM
import test_gpu_resync as RS
import test_gpu_row_index as RI
import wire_rewrite as W
from util import assert_columns_equal

pytestmark = pytest.mark.gpu

BA = TFR_RT_BYTE_ARRAY


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


# ---------------------------------------------------------------------------------------------
# corpora
# ---------------------------------------------------------------------------------------------
def image_schema():
    return StructType([StructField("id", LongType()), StructField("label", FloatType()), StructField("name", StringType()),
                       StructField("image", BinaryType())])


def image_corpus(n, size, seed, jitter=0, outliers=()):
    """Examples with one BytesList 'image' of `size` (+- jitter) bytes next to scalar fields; rows in `outliers` get 200 KB"""
    R = random.Random(seed)
    sch = image_schema()
    pay = []
    for i in range(n):
        sz = 200_000 if i in outliers else size + (R.randint(-jitter, jitter) if jitter else 0)
        row = [R.randint(-2**40, 2**40), R.random(), f"rec-{i}-{'xé漢𝄞'[R.randint(0, 3)] * R.randint(0, 20)}", R.randbytes(max(sz, 1))]
        pay.append(pyref.serialize_example_bytes(sch, row))
    return sch, b"".join(pyref.frame_fast(p) for p in pay)


def embed_schema(elem):
    return StructType([StructField("id", LongType()), StructField("emb", ArrayType(elem)), StructField("tag", StringType())])


def embed_corpus(n, length, seed, elem=FloatType(), ragged=False):
    R = random.Random(seed)
    sch = embed_schema(elem)
    pay = []
    for i in range(n):
        L = R.randint(length // 2, length) if ragged else length
        if isinstance(elem, LongType):
            vals = [R.randint(-2**62, 2**62) if R.random() < 0.3 else R.randint(0, 300) for _ in range(L)]
        else:
            vals = list(np.frombuffer(np.random.default_rng(seed + i).standard_normal(L).astype(np.float32).tobytes(), np.float32).astype(float))
        pay.append(pyref.serialize_example_bytes(sch, [i, vals, f"t{i}"]))
    return sch, b"".join(pyref.frame_fast(p) for p in pay)


def bytes_corpus(n, lo, hi, seed):
    R = random.Random(seed)
    return b"".join(pyref.frame_fast(R.randbytes(R.randint(lo, hi))) for _ in range(n))


def byte_array_schema():
    return StructType([StructField("value", BinaryType())])


def delta(s0, s1):
    return {k: s1[k] - s0[k] for k in s0}


def check_decode(native, oracle, sch, data, rt=0):
    """a fresh decoder: one synchronous decode == the oracle (info, host columns, rows); returns its stats"""
    want = oracle.decode(data, sch, rt)
    dec = native.Decoder(sch, rt)
    try:
        b, used = dec.decode(data)
        assert used == want.info["consumed_bytes"]
        for k in ("n_rows", "error_code", "error_row", "error_field"):
            assert b.info[k] == want.info[k], (k, b.info[k], want.info[k])
        assert_columns_equal(b.to_host(), want.columns, None, "sync decode")
        check_batch(native, oracle, b, data, sch, rt)
        b.release()
        return dec.stats()
    finally:
        dec.close()


def stream(native, oracle, sch, blocks, rt=0, on_device=False):
    """every block submitted in turn (pipelined once learned), each checked against the oracle; returns the stats' delta"""
    import torch
    dec = native.Decoder(sch, rt)
    try:
        s0 = dec.stats()
        for data in blocks:
            src = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda() if on_device else data
            b = dec.submit(src)
            want = oracle.decode(data, sch, rt)
            assert b.info["n_rows"] == want.info["n_rows"]
            assert_columns_equal(b.to_host(), want.columns, None, "pipelined")
            b.release()
        return delta(s0, dec.stats())
    finally:
        dec.close()


def expect_of(oracle, data, sch, rt=0):
    """the oracle's decode of a clean block as a drop-mode Expect (for D.check_rows)"""
    w = oracle.decode(data, sch, rt)
    return D.Expect(w.columns, {k: w.info[k] for k in ("n_rows", "n_records", "consumed_bytes", "error_code", "error_row", "error_field")}, [])


def assert_contract(d, n_blocks, large=True):
    assert d["speculative_submits"] == n_blocks - 1, d      # after the learning batch every submit is speculative
    assert d["speculative_redone"] == 0 and d["general_path_batches"] == 0 and d["rows_async_rebuilt"] == 0, d
    if large:                                               # (records that fit a tile keep the tile kernels)
        assert d["large_record_batches"] == n_blocks, d


# ---------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", [8 << 10, (64 << 10) - 1, (64 << 10) + 1, 1 << 20, 4 << 20])
def test_image_examples(native, oracle, size):
    n = max(6, min(40, (24 << 20) // size))
    sch, data = image_corpus(n, size, seed=size)
    st = check_decode(native, oracle, sch, data)
    assert st["general_path_batches"] == 0 and st["large_record_batches"] == 1, st


@pytest.mark.parametrize("on_device", [False, True])
def test_image_stream_contract(native, oracle, on_device):
    blocks = [image_corpus(96, 16 << 10, seed=10 + k, jitter=2000)[1] for k in range(5)]
    d = stream(native, oracle, image_schema(), blocks, on_device=on_device)
    assert_contract(d, len(blocks))


@pytest.mark.parametrize("elem", [FloatType(), DoubleType(), LongType(), IntegerType()], ids=str)
@pytest.mark.parametrize("ragged", [False, True])
def test_embeddings(native, oracle, elem, ragged):
    for length in (2048, 262_144):
        n = 80 if length == 2048 else 4
        blocks = [embed_corpus(n, length, seed=length + k, elem=elem, ragged=ragged)[1] for k in range(3)]
        sch = embed_schema(elem)
        check_decode(native, oracle, sch, blocks[0])
        d = stream(native, oracle, sch, blocks)
        if length == 2048:                                  # (four records are too few to learn from)
            assert_contract(d, len(blocks), large=len(blocks[0]) / n > 7800)


def test_byte_array(native, oracle):
    sch = byte_array_schema()
    for lo, hi, n in ((8 << 10, 64 << 10, 100), (1 << 20, 8 << 20, 6)):
        blocks = [bytes_corpus(n, lo, hi, seed=lo + k) for k in range(3)]
        st = check_decode(native, oracle, sch, blocks[0], BA)
        assert st["large_record_batches"] == 1, st
        d = stream(native, oracle, sch, blocks, BA)
        if n > 64:
            assert_contract(d, len(blocks))


def test_mostly_small_with_outliers(native, oracle):
    """rare 200 KB records among 1.2 KB ones: the largest record is far above 8x the mean, so these batches stay on the general
    path (measured faster there); the results are the oracle's either way"""
    blocks = [image_corpus(400, 1200, seed=50 + k, jitter=300, outliers={17 + k, 301})[1] for k in range(4)]
    d = stream(native, oracle, image_schema(), blocks)
    assert d["large_record_batches"] == 0, d
    # outliers of about 5x the mean: the large-record kernel, pipelined
    blocks = [image_corpus(400, 40_000, seed=60 + k, jitter=1000, outliers={17 + k, 301})[1] for k in range(4)]
    d = stream(native, oracle, image_schema(), blocks)
    assert_contract(d, len(blocks))


def test_odd_address_and_streaming_carry(native, oracle):
    import torch
    sch, data = image_corpus(70, 20_000, seed=3, jitter=5000)
    want = oracle.decode(data, sch)
    dec = native.Decoder(sch)
    try:
        buf = torch.zeros(len(data) + 1, dtype=torch.uint8, device="cuda")
        buf[1:] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        b, _ = dec.decode((buf.data_ptr() + 1, len(data), 1))
        assert_columns_equal(b.to_host(), want.columns, None, "odd address")
        b.release()
    finally:
        dec.close()
    # blocks of 7 KB, smaller than one record: the carry grows until a record is whole
    dec = native.Decoder(sch)
    try:
        rows, carry, pos = 0, b"", 0
        while True:
            blk = carry + data[pos:pos + 7000]
            pos += 7000
            final = pos >= len(data)
            b, used = dec.decode(blk, is_final=final)
            if b.info["n_rows"]:
                w = oracle.decode(blk[:used], sch)
                assert_columns_equal(b.to_host(), w.columns, None, "streamed block")
            rows += b.info["n_rows"]
            b.release()
            carry = blk[used:]
            if final:
                break
        assert rows == 70
    finally:
        dec.close()


@pytest.mark.parametrize("flags", [D.DROP], ids=["drop"])
@pytest.mark.parametrize("damage", ["crc", "kind", "truncated"])
def test_malformed(native, oracle, flags, damage):
    sch = image_schema()
    R = random.Random(7)
    pays = []
    for i in range(40):
        row = [i, 0.5, f"r{i}", R.randbytes(12_000)]
        p = pyref.serialize_example_bytes(sch, row)
        if damage == "kind" and i == 11:
            p = pyref.serialize_example_bytes(StructType([StructField("id", LongType()), StructField("label", FloatType()),
                                                          StructField("name", StringType()), StructField("image", LongType())]),
                                              [i, 0.5, f"r{i}", 5])
        pays.append(p)
    frames = [bytearray(pyref.frame_fast(p)) for p in pays]
    if damage == "crc":
        frames[9][500] ^= 0x40
    data = bytes(b"".join(frames))
    if damage == "truncated":
        data = data[:-3000]
    D.check_fresh(native, oracle, data, sch, 0, flags=flags, what=damage)
    # FAILFAST: the error at the right record, the rows in front of it
    want = oracle.decode(data, sch)
    dec = native.Decoder(sch)
    try:
        b, _ = dec.decode(data)
        for k in ("n_rows", "error_code", "error_row", "error_field"):
            assert b.info[k] == want.info[k], (k, b.info[k], want.info[k])
        b.release()
    finally:
        dec.close()


def test_repeated_features_message(native, oracle):
    """a record whose Features message comes twice (protobuf merges them; the key written again wins): the parse the large-record
    kernel shares with the general path takes it, with the oracle's result"""
    import wire_rewrite as W
    sch = image_schema()
    R = random.Random(11)
    rows = [[i, 0.25, f"n{i}", R.randbytes(10_000)] for i in range(80)]
    clean = [pyref.serialize_example_bytes(sch, r) for r in rows]
    learn = b"".join(pyref.frame_fast(p) for p in clean)
    # a non-canonical but equivalent record: the map entry of 'id' written twice (last wins) in record 5
    extra = W.entry(b"id", W.feature(W.kind_of(LongType()), W.elems_of(W.kind_of(LongType()), [123])))
    payloads = list(clean)
    payloads[5] = pyref.ld(1, extra) + clean[5]              # a second Features occurrence in front: merged, non-canonical
    data = b"".join(pyref.frame_fast(p) for p in payloads)
    dec = native.Decoder(sch)
    try:
        b, _ = dec.decode(learn)
        b.release()
        s0 = dec.stats()
        b = dec.submit(data)
        want = oracle.decode(data, sch)
        assert_columns_equal(b.to_host(), want.columns, None, "repeated Features")
        d = delta(s0, dec.stats())
        assert d["general_path_batches"] == 0 and d["large_record_batches"] == 1, d
        b.release()
    finally:
        dec.close()


def test_rows_async_and_partition_rows(native, oracle):
    """UnsafeRows enqueued at submit time (counter [7] rises, none rebuilt), with and without partition values"""
    sch = image_schema()
    blocks = [image_corpus(96, 16 << 10, seed=30 + k, jitter=2000)[1] for k in range(5)]
    for part in (None, D.PART):                             # (a batch's rows are built with one partition row)
        pr = None if part is None else (P.partition_row(*part), P.var_flags(part[0]))    # (types, values) -> the ABI's row
        dec = native.Decoder(sch)
        try:
            s0 = dec.stats()
            for k, data in enumerate(blocks):
                b = dec.submit(data)
                b.unsafe_rows_async(to_host=True, partition=pr)
                want = None if part is None else D.want_rows(sch, expect_of(oracle, data, sch), part)
                RP.check_async(native, oracle, b, data, sch, want_rows=want, partition=pr)
                b.release()
            d = delta(s0, dec.stats())
            # block 0 (learning) teaches the row sizes when its rows are built, before block 1 is submitted: every later block's
            # rows are enqueued at submit time
            assert d["rows_async"] == len(blocks) - 1 and d["rows_async_rebuilt"] == 0, d
            assert_contract(d, len(blocks))
        finally:
            dec.close()


def test_generated_position_fields(native, oracle):
    """row index and record offset of every row (Spark's _metadata.row_index) on pipelined large-record batches"""
    sch = image_schema()
    gsch, gi, didx = RI.add_generated(sch, 0, "middle")
    dec = native.Decoder(gsch)
    try:
        s0 = dec.stats()
        entry, offset = 0, 0
        for k in range(4):
            data = image_corpus(80, 12 << 10, seed=40 + k, jitter=3000)[1]
            b = dec.submit(data, first_entry=entry, first_offset=offset)
            cols = b.to_host()
            want = oracle.decode(data, sch)
            assert_columns_equal([cols[i] for i in didx], want.columns, None, f"block {k} data")
            RI.check_positions(cols, gi, RI.expect(oracle, data, sch, 0, A.TFR_F_DEFAULT, base=(entry, offset)), f"block {k}")
            entry += want.info["n_rows"]; offset += len(data)
            b.release()
        assert_contract(delta(s0, dec.stats()), 4)
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# wire forms the large-record kernel must not take: CRC-valid, protobuf-valid rewrites of one record after the decoder has
# learned its shapes.  The result is the oracle's, and the batch is redone.
# ---------------------------------------------------------------------------------------------
def wire_schema():
    return StructType([StructField("id", LongType()), StructField("s", StringType()), StructField("tags", ArrayType(StringType())),
                       StructField("ints", ArrayType(LongType())), StructField("blob", BinaryType())])


def _feat_bytes(elems, tag=b"\x0a"):
    return pyref.ld(1, b"".join(tag + pyref.varint(len(e)) + e for e in elems))


def _feat_ints(vals, pad=0):
    packed = b"".join(pyref.varint(v) for v in vals)
    return pyref.ld(3, W.ld_ov(1, packed, pad) if pad else pyref.ld(1, packed))


def wire_record(R, i, ragged, rewrite=None):
    s = b"abcdef" if not ragged else b"abcdef"[:R.randint(1, 6)] + "é".encode()
    tags = [b"tag", "ü-tag".encode(), b"x" * R.randint(1, 30)]
    ints = [R.randint(0, 2**40) for _ in range(R.randint(1024, 2048) if ragged else 2048)]
    fs = {"id": pyref.ld(3, pyref.ld(1, pyref.varint(i))), "s": _feat_bytes([s]), "tags": _feat_bytes(tags), "ints": _feat_ints(ints),
          "blob": _feat_bytes([R.randbytes(6000)])}
    if rewrite == "overlong_plen":
        fs["ints"] = _feat_ints(ints, pad=4)
    elif rewrite == "overlong_elem_tag":
        fs["tags"] = _feat_bytes(tags, tag=b"\x8a\x00")
    elif rewrite == "overlong_str_len":
        fs["s"] = pyref.ld(1, b"\x0a" + W.ov(len(s), 2) + s)
    elif rewrite == "surrogate_scalar":                     # 3 bytes in, U+FFFD (3 bytes) out: the length does not change
        fs["s"] = _feat_bytes([s[:-3] + b"\xed\xa0\x80" if len(s) >= 3 else b"\xed\xa0\x80"])
    elif rewrite == "truncated_4byte_in_list":               # F1 80 80 41 -> U+FFFD 'A': 4 bytes either way
        fs["tags"] = _feat_bytes(tags[:1] + [b"\xf1\x80\x80\x41"] + tags[2:])
    return pyref.ld(1, b"".join(pyref.map_entry(k.encode(), v) for k, v in fs.items()))


REWRITES = ["overlong_plen", "overlong_elem_tag", "overlong_str_len", "surrogate_scalar", "truncated_4byte_in_list"]


@pytest.mark.parametrize("ragged", [False, True], ids=["uniform", "ragged"])
@pytest.mark.parametrize("rewrite", REWRITES)
def test_non_canonical_and_malformed_utf8_flag_and_redo(native, oracle, rewrite, ragged):
    sch = wire_schema()
    R = random.Random(REWRITES.index(rewrite) * 2 + ragged)
    learn = [b"".join(pyref.frame_fast(wire_record(R, i, ragged)) for i in range(80)) for _ in range(2)]
    bad = b"".join(pyref.frame_fast(wire_record(R, i, ragged, rewrite if i == 7 else None)) for i in range(80))
    dec = native.Decoder(sch)
    try:
        for data in learn:
            b = dec.submit(data)
            assert_columns_equal(b.to_host(), oracle.decode(data, sch).columns, None, "learning")
            b.release()
        s0 = dec.stats()
        assert s0["large_record_batches"] == 2 and s0["speculative_submits"] == 1, s0
        b = dec.submit(bad)
        want = oracle.decode(bad, sch)
        assert want.info["error_code"] == 0
        assert_columns_equal(b.to_host(), want.columns, None, rewrite)
        check_batch(native, oracle, b, bad, sch)
        b.release()
        d = delta(s0, dec.stats())
        assert d["speculative_submits"] == 1 and d["speculative_redone"] == 1, d
    finally:
        dec.close()


@pytest.mark.parametrize("mode", ["drop", "drop_resync", "perm", "perm_resync", "perm_nocol"])
@pytest.mark.parametrize("damage", ["crc", "kind", "truncated", "lencrc"])
def test_malformed_after_learning(native, oracle, mode, damage):
    """a damaged block submitted once the decoder is pipelined, in every tolerant mode: the oracle-derived expectation"""
    flags = {"drop": D.DROP, "drop_resync": D.DROP | A.TFR_F_RESYNC, "perm": PM.PERM, "perm_resync": PM.PERM | A.TFR_F_RESYNC,
             "perm_nocol": PM.PERM}[mode]
    pos = "middle" if mode in ("perm", "perm_resync") else None
    sch = image_schema()
    R = random.Random(5)
    clean = image_corpus(80, 12_000, seed=77)[1]
    frames = [bytearray(pyref.frame_fast(pyref.serialize_example_bytes(sch, [i, 0.5, f"r{i}", R.randbytes(12_000)]))) for i in range(40)]
    if damage == "crc":
        frames[9][500] ^= 0x40
    elif damage == "kind":
        frames[11] = bytearray(pyref.frame_fast(pyref.example({"id": pyref.int64_feature(1), "image": pyref.int64_feature(5)}).SerializeToString()))
    elif damage == "lencrc":
        frames[13][9] ^= 0x01
    data = bytes(b"".join(frames))
    if damage == "truncated":
        data = data[:-3000]
    exp = None
    for part in (None, D.PART):                             # (a batch's rows are built with one partition row)
        full, cf, dec = RS.decoder(native, sch, 0, flags, pos)
        try:
            if exp is None:
                if flags & A.TFR_F_RESYNC:
                    exp = RS.expected(oracle, data, full, 0, flags, True, cf)
                elif flags & A.TFR_F_PERMISSIVE:
                    exp = PM.expected(oracle, data, full, 0, flags, cf)
                else:
                    exp = D.expected(oracle, data, full, 0, flags)
            for _ in range(2):                                  # learning, then one pipelined clean block
                b = dec.submit(clean)
                b.wait()
                b.release()
            assert dec.stats()["large_record_batches"] == 2 and dec.stats()["speculative_submits"] == 1, dec.stats()
            b = dec.submit(data)
            what = f"{mode} {damage}"
            if part is not None:
                D.check_rows(b, full, exp, part, what + " with partition values")
            elif flags & A.TFR_F_RESYNC:
                RS.check_batch(b, full, exp, what)
            else:
                D.check_info(b, exp, what)
                assert_columns_equal(b.to_host(), exp.columns, None, what)
                D.check_rows(b, full, exp, None, what)
            b.release()
        finally:
            dec.close()
