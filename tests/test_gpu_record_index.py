"""The record index on the GPU (include/tfrgpu.h, RECORD INDEX; the DataSource option recordIndex=true).

  1. Build: golden files and seeded Example / SequenceExample / ByteArray files, from host and from device input, in blocks
     cut at random places, for strides from 16 B to 1 MiB: the index bytes equal tests/record_index.py's byte for byte.  A
     framing error fails the build at its file offset.
  2. Writer: recordIndex=true writes buildIndex's index, and the same data bytes as a write without the option.
  3. Splits: the rows of all splits of a file, concatenated, equal the whole-file read with row_index and record_offset, in
     FAILFAST on clean files and DROPMALFORMED / PERMISSIVE on files with record errors; each clean split against the oracle.
  4. Mismatch: a shifted checkpoint, an entry off by one and another file's index raise TFR_E_INDEX_MISMATCH, and never
     hand out a row the whole-file read does not.
  5. Embedded frames: frame_embedded_tfrecords.tfrecord split at every byte offset reads exactly the outer records."""
import os
import random
import struct

import numpy as np
import pytest

import record_index as RX
import resync_walk as RW
from oracle import corpus, oracle, pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200 import io as tio
from spark_tfrecord_b200.sqltypes import (ArrayType, BinaryType, FloatType, LongType, StringType, StructField, StructType,
                                          byte_array_schema)

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RI, RO = "_tmp_metadata_row_index", "_tmp_metadata_record_offset"
STRIDES = [16, 64, 1024, 1 << 14, 1 << 20]


def golden_files():
    return sorted(f for f in os.listdir(GOLDEN) if f.endswith(".tfrecord"))


def example_file(n, seed):
    schema, cols = corpus.cfg2_columns(n, seed=seed, n_int=4, n_float=2, n_bytes=2)
    data, rc, _ = oracle.encode(cols, schema)
    assert rc == 0
    return bytes(data), schema


def seq_file(n, seed):
    schema, cols = corpus.cfg4_columns(n, seed=seed, mean_steps=4)
    data, rc, _ = oracle.encode(cols, schema, 1)
    assert rc == 0
    return bytes(data), schema


def bytearray_file(n, seed):
    rng = random.Random(seed)
    return b"".join(pyref.frame(rng.randbytes(rng.choice([0, 1, 7, 100, 3000, 70000]))) for _ in range(n))


def build(data, stride, cuts=(), device=False):
    """the index of `data` streamed in blocks ending at `cuts` (a block that consumes nothing grows by the next cut)"""
    idx = _native.Indexer(stride)
    try:
        cuts = sorted(c for c in set(cuts) if 0 < c < len(data)) + [len(data)]
        pos, i = 0, 0
        while True:
            while cuts[i] < pos or (cuts[i] == pos and pos < len(data)):
                i += 1
            stop = cuts[i]
            final = stop == len(data)
            blk = data[pos:stop]
            if device:
                import torch
                t = torch.tensor(np.frombuffer(blk, dtype=np.uint8).copy(), device="cuda") if blk else torch.empty(0, dtype=torch.uint8, device="cuda")
                used = idx.update(t, final)
            else:
                used = idx.update(blk, final)
            if final:
                assert used == len(blk)
                break
            if used == 0:
                i += 1
            pos += used
        return idx.result()
    finally:
        idx.close()


# ---------------------------------------------------------------------------------------------
# 1. build
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", golden_files())
def test_golden_files(name):
    data = open(os.path.join(GOLDEN, name), "rb").read()
    try:
        want = RX.index_bytes(data, 16)
    except RX.FramingError as fe:
        with pytest.raises(_native.IOException) as e:
            build(data, 16)
        assert e.value.code == fe.code and f"file offset {fe.offset} " in str(e.value)
        return
    for stride in (16, 32, 1 << 20):
        assert build(data, stride) == RX.index_bytes(data, stride), stride
    assert build(data, 16, cuts=range(0, len(data), 7)) == want


@pytest.mark.parametrize("kind", ["example", "seq", "bytes"])
@pytest.mark.parametrize("device", [False, True])
def test_random_files_random_cuts(kind, device):
    rng = random.Random(f"{kind}-{device}")
    data = {"example": lambda: example_file(3000, 5)[0], "seq": lambda: seq_file(500, 6)[0], "bytes": lambda: bytearray_file(300, 7)}[kind]()
    offs = RX.frames(data)
    for stride in STRIDES:
        cuts = [rng.randrange(len(data)) for _ in range(rng.choice([0, 1, 5, 40]))]
        got = build(data, stride, cuts, device)
        assert got == RX.index_bytes(data, stride), (kind, stride, cuts)
        assert struct.unpack_from("<Q", got, 16)[0] == len(offs)


def test_framing_error_fails_at_its_offset():
    data = bytearray(bytearray_file(50, 9))
    offs = RX.frames(bytes(data))
    data[offs[31] + 9] ^= 0x10                  # the length CRC of frame 31
    for cuts in ([], [offs[30] + 3], list(range(0, len(data), 997))):
        with pytest.raises(_native.IOException) as e:
            build(bytes(data), 64, cuts)
        assert e.value.code == A.TFR_E_CRC_LENGTH and f"file offset {offs[31]} " in str(e.value)
    with pytest.raises(_native.IOException) as e:                     # a truncated file
        build(bytes(data[:offs[40] + 20]), 64)
    assert e.value.code == A.TFR_E_CRC_LENGTH                          # (frame 31 comes first)
    clean = bytearray_file(50, 9)
    with pytest.raises(_native.IOException) as e:
        build(clean[:RX.frames(clean)[40] + 20], 64)
    assert e.value.code == A.TFR_E_TRUNCATED and f"file offset {RX.frames(clean)[40]} " in str(e.value)


def test_result_before_final_and_update_after_failure():
    idx = _native.Indexer(16)
    with pytest.raises(_native.TfrError) as e:
        idx.result()
    assert e.value.code == A.TFR_E_INVALID_ARG
    bad = bytearray(pyref.frame(b"abc"))
    bad[9] ^= 1
    with pytest.raises(_native.IOException):
        idx.update(bytes(bad), True)
    with pytest.raises(_native.IOException):
        idx.result()
    idx.close()


def test_seek_against_the_rule():
    data = bytearray_file(200, 11)
    offs = RX.frames(data)
    for stride in (16, 256, 4096):
        n, _, ck = tio.parse_index(RX.index_bytes(data, stride), len(data))
        idx = _native.Indexer(stride)
        try:
            for t in sorted(set([0, len(data) - 1] + [random.Random(t0).randrange(len(data)) for t0 in range(60)] +
                                [o + d for o in offs[:20] for d in (-1, 0, 1, 12)])):
                if not 0 <= t < len(data):
                    continue
                off, ent = int(ck[t // stride][0]), int(ck[t // stride][1])
                got = idx.seek(data[off:min(len(data), t + 12)] if t + 12 > off else b"", ent, off, t)
                assert got == RX.seek(offs, len(data), t), (stride, t)
        finally:
            idx.close()


# ---------------------------------------------------------------------------------------------
# 2. writer
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [0, 1, 5000])
def test_writer_index_equals_build_index(tmp_path, rows):
    schema = StructType([StructField("id", LongType(), False), StructField("s", StringType(), True),
                         StructField("v", ArrayType(FloatType()), True)])
    data = [(i, None if i % 7 == 0 else "x" * (i % 50), [float(i)] * (i % 9)) for i in range(rows)]
    ds = tio.DefaultSource()
    ds.save(str(tmp_path / "plain"), schema, data)
    tio.TFRecordOutputWriter.FLUSH_ROWS, keep = 777, tio.TFRecordOutputWriter.FLUSH_ROWS   # several flushes, each indexed
    try:
        ds.save(str(tmp_path / "indexed"), schema, data, {"recordIndex": "true"})
    finally:
        tio.TFRecordOutputWriter.FLUSH_ROWS = keep
    p0, p1 = str(tmp_path / "plain" / "part-00000.tfrecord"), str(tmp_path / "indexed" / "part-00000.tfrecord")
    assert open(p0, "rb").read() == open(p1, "rb").read()
    assert not os.path.exists(tio.index_path(p0))
    written = open(tio.index_path(p1), "rb").read()
    assert written == RX.index_bytes(open(p1, "rb").read(), tio.RECORD_INDEX_STRIDE)
    os.rename(tio.index_path(p1), str(tmp_path / "w"))
    assert open(ds.buildIndex(p1), "rb").read() == written
    assert ds.isSplitable({"recordIndex": "true"}, p1)
    assert sorted(os.listdir(tmp_path / "indexed")) == ["_SUCCESS", "_part-00000.tfrecord.tfrindex", "part-00000.tfrecord"]
    assert ds.load(str(tmp_path / "indexed"), schema) == ds.load(str(tmp_path / "plain"), schema)


# ---------------------------------------------------------------------------------------------
# 3. splits
# ---------------------------------------------------------------------------------------------
def with_positions(schema):
    return StructType(list(schema.fields) + [StructField(RI, LongType(), False), StructField(RO, LongType(), False)])


def read(path, schema, options, start=0, length=None, block_bytes=None):
    return list(tio.TFRecordFileReader.readFile(None, options, tio.PartitionedFile(path, start, length), schema,
                                                block_bytes=block_bytes))


def split_points(rng, data, offs, n):
    pts = {0, len(data)}
    for _ in range(n):
        r = rng.random()
        if r < 0.3:
            pts.add(rng.choice(offs))                                       # exactly on a boundary
        elif r < 0.5:
            pts.add(min(len(data), rng.choice(offs) + rng.randrange(1, 12)))   # inside a header
        else:
            pts.add(rng.randrange(len(data) + 1))
    k = rng.randrange(len(data))
    pts.update((k, k + 1, k + 2))                                           # 1-byte splits
    return sorted(p for p in pts if 0 <= p <= len(data))


def check_splits(path, schema, options, data, pts, whole):
    got = []
    for s, e in zip(pts, pts[1:]):
        got += read(path, schema, options, s, e - s, block_bytes=4096)
    assert got == whole


def damaged_example_file(seed):
    """an Example file with record errors: payload CRC flips and CRC-valid frames whose payload is not a protobuf"""
    data, schema = example_file(1500, seed)
    offs = RX.frames(data) + [len(data)]
    rng = random.Random(seed)
    out = bytearray()
    for i in range(len(offs) - 1):
        fr = bytearray(data[offs[i]:offs[i + 1]])
        r = rng.random()
        if r < 0.03:
            fr[12 + rng.randrange(len(fr) - 16)] ^= 0x40                   # TFR_E_CRC_DATA
        elif r < 0.06:
            fr = bytearray(pyref.frame(b"\x0a\xff\xff\xff\xff\x0f" + bytes(fr[12:20])))   # TFR_E_MALFORMED_PROTO
        out += fr
    return bytes(out), schema


@pytest.mark.parametrize("kind", ["example", "seq", "bytes"])
def test_splits_concatenate_to_the_whole_file_failfast(tmp_path, kind):
    rng = random.Random(kind)
    if kind == "bytes":
        data, schema, opts = bytearray_file(400, 3), byte_array_schema(), {"recordType": "ByteArray"}
        schema = StructType([StructField(RI, LongType(), False), StructField(RO, LongType(), False)])
    else:
        data, schema = example_file(4000, 21) if kind == "example" else seq_file(600, 22)
        opts = {} if kind == "example" else {"recordType": "SequenceExample"}
        schema = with_positions(schema)
    p = str(tmp_path / "f.tfrecord")
    open(p, "wb").write(data)
    whole = read(p, schema, opts)
    offs = RX.frames(data)
    assert [r[-2:] for r in whole] == [(i, o) for i, o in enumerate(offs)]
    on = {**opts, "recordIndex": "true"}
    for stride in (16, 4096, 1 << 20):
        open(tio.index_path(p), "wb").write(build(data, stride))
        assert tio.DefaultSource().isSplitable(on, p)
        check_splits(p, schema, on, data, split_points(rng, data, offs, 30), whole)
    # each split against the oracle (the frames of [offset(s), offset(e)))
    if kind != "bytes":
        plain = StructType(schema.fields[:-2])
        pts = split_points(rng, data, offs, 12)
        for s, e in zip(pts, pts[1:]):
            rows = read(p, schema, on, s, e - s)
            i0, i1 = RX.seek(offs, len(data), s)[0], RX.seek(offs, len(data), e)[0]
            assert [r[-2] for r in rows] == list(range(i0, i1))
            if i1 > i0:
                lo, hi = offs[i0], (offs[i1] if i1 < len(offs) else len(data))
                want = oracle.decode(data[lo:hi], plain, 0 if kind == "example" else 1)
                assert want.info["error_code"] == 0
                assert [r[:-2] for r in rows] == list(want.rows())


@pytest.mark.parametrize("mode", ["DROPMALFORMED", "PERMISSIVE", "FAILFAST"])
def test_splits_with_record_errors(tmp_path, mode):
    data, schema = damaged_example_file(31)
    if mode == "PERMISSIVE":
        schema = StructType(list(schema.fields) + [StructField("_corrupt_record", BinaryType(), True)])
    schema = with_positions(schema)
    p = str(tmp_path / "d.tfrecord")
    open(p, "wb").write(data)
    opts = {"mode": mode}
    offs = RX.frames(data)
    open(tio.index_path(p), "wb").write(build(data, 512))
    on = {**opts, "recordIndex": "true"}
    rng = random.Random(mode)
    if mode != "FAILFAST":
        whole = read(p, schema, opts)
        assert len(whole) < len(offs) if mode == "DROPMALFORMED" else len(whole) == len(offs)
        for _ in range(3):
            check_splits(p, schema, on, data, split_points(rng, data, offs, 25), whole)
        return
    # FAILFAST raises at the split's first failing record, after the rows in front of it
    with pytest.raises(_native.TfrError) as e0:
        read(p, schema, opts)
    pts = split_points(rng, data, offs, 25)
    for s, e in zip(pts, pts[1:]):
        rows = []
        try:
            for r in tio.TFRecordFileReader.readFile(None, on, tio.PartitionedFile(p, s, e - s), schema, block_bytes=4096):
                rows.append(r)
        except _native.TfrError as err:
            assert type(err) is type(e0.value) or isinstance(err, _native.IOException)
        i0 = RX.seek(offs, len(data), s)[0]
        assert [r[-2] for r in rows] == list(range(i0, i0 + len(rows)))
        assert [r[-1] for r in rows] == offs[i0:i0 + len(rows)]


# ---------------------------------------------------------------------------------------------
# 4. mismatch
# ---------------------------------------------------------------------------------------------
def corrupt_index(raw, k, d_off=0, d_ent=0):
    b = bytearray(raw)
    o, e = struct.unpack_from("<QQ", b, 32 + 16 * k)
    struct.pack_into("<QQ", b, 32 + 16 * k, o + d_off, e + d_ent)
    return bytes(b)


@pytest.mark.parametrize("how", ["shift", "entry", "other_file"])
def test_mismatch_raises_and_never_returns_a_wrong_row(tmp_path, how):
    data, schema = example_file(2000, 41)
    schema = with_positions(schema)
    p = str(tmp_path / "m.tfrecord")
    open(p, "wb").write(data)
    whole = {repr(r) for r in read(p, schema, {})}
    offs = RX.frames(data)
    stride = 1024
    raw = build(data, stride)
    n_ck = (len(raw) - 32) // 16
    if how == "other_file":
        # another file's checkpoints under a header that claims this file's size (a plain other index fails the size check)
        o_offs = [o for o in RX.frames(bytearray_file(400, 43)) if o < len(data)]
        ck = RX.checkpoints(o_offs, len(data), stride)
        bad = [RX.HEADER.pack(RX.MAGIC, len(data), len(o_offs), stride) + b"".join(struct.pack("<QQ", o, e) for o, e in ck)]
    elif how == "shift":
        bad = [corrupt_index(raw, k, d_off=d) for k in (3, n_ck // 2, n_ck - 2) for d in (1, -1)]
    else:
        bad = [corrupt_index(raw, k, d_ent=d) for k in (3, n_ck // 2, n_ck - 2) for d in (1, -1)]
    on = {"recordIndex": "true"}
    raised = 0
    ks = (3, n_ck // 2, n_ck - 2)
    for b in bad:
        open(tio.index_path(p), "wb").write(b)
        # splits that start at a damaged checkpoint, splits that end at one, and a few others
        for s in sorted({k * stride for k in ks} | {(k - 1) * stride for k in ks} | {0, 7 * stride + 5, len(data) - stride}):
            rows = []
            try:
                for r in tio.TFRecordFileReader.readFile(None, on, tio.PartitionedFile(p, s, stride), schema):
                    rows.append(r)
            except _native.IOException as err:
                assert err.code in (A.TFR_E_INDEX_MISMATCH, A.TFR_E_CRC_LENGTH), err
                raised += 1
            assert {repr(r) for r in rows} <= whole, (how, s)
    assert raised >= len(bad)


# ---------------------------------------------------------------------------------------------
# 5. embedded frames
# ---------------------------------------------------------------------------------------------
def test_embedded_frames_split_at_every_offset(tmp_path):
    data = open(os.path.join(GOLDEN, "frame_embedded_tfrecords.tfrecord"), "rb").read()
    p = str(tmp_path / "e.tfrecord")
    open(p, "wb").write(data)
    open(tio.index_path(p), "wb").write(build(data, 16))
    schema = StructType([StructField(RI, LongType(), False), StructField(RO, LongType(), False)])
    opts = {"recordType": "ByteArray"}
    whole = read(p, schema, opts)
    offs = RX.frames(data)
    assert [r[1:] for r in whole] == [(i, o) for i, o in enumerate(offs)]
    on = {**opts, "recordIndex": "true"}
    # the seek of every byte offset finds the outer frame a split starting there begins with
    n, stride, ck = tio.parse_index(open(tio.index_path(p), "rb").read(), len(data))
    idx = _native.Indexer(stride)
    try:
        for t in range(len(data) + 1):
            if t == len(data):
                got = (n, len(data))
            else:
                off, ent = int(ck[t // stride][0]), int(ck[t // stride][1])
                got = idx.seek(data[off:min(len(data), t + 12)] if t + 12 > off else b"", ent, off, t)
            assert got == RX.seek(offs, len(data), t), t
    finally:
        idx.close()
    # and the reads themselves, cut around every position whose header verifies (outer and embedded frames) and elsewhere
    near = {q + d for q in range(len(data) - 12) if RW.header_ok(data, q) for d in (0, 1)}
    near |= {q + d for q in offs for d in (-1, 0, 1, 12)}
    for s in sorted(t for t in near | set(range(0, len(data) + 1, 4099)) if 0 <= t <= len(data)):
        got = read(p, schema, on, 0, s) + read(p, schema, on, s, len(data) - s)
        assert got == whole, s
