"""GPU tests of every CRC-32C routine at the lengths, start offsets and bit flips where its split of a payload changes
(crc_corpus.py has the sets).  Each routine is reached through the path that runs it, and the test checks through the
decoder's stats that it was that path:

  general     crc_warp (decode.cuh), TFR_DISABLE_FAST
  tile_4_1    decode tile, one CRC warp, fixed slots (records up to 625 B)
  tile_12_3   decode tile, three CRC warps, fixed slots (a record above 625 B in the batch)
  packed      decode tile, three CRC warps, packed layout of a pipelined submit: one record of 12-38 KB among small ones,
              whose leading warps shift their CRC by 512 chunks or more (past the xp16 table)
  bytes_4_2 / bytes_8_4   ByteArray decode kernels
  large_example / large_bytes   large_crc (large.cuh), and one ByteArray record of 48 MiB
  infer       schema inference (crc_warp), resync   the resync scan (crc_warp)
and the encoders: the Example encode tile, the general emit kernel, the ByteArray encode kernels.

Clean batches must equal the oracle and stay on their path; a batch with one damaged record must give the oracle's error
at that record, and the clean batch after it must be on the path again.  A wrong CRC on a fast decode path is invisible in
the output (the batch is redone on the general path), so the path assertions are what catches a false mismatch."""
import os
import random
import struct

import numpy as np
import pytest

import crc_corpus as K
from oracle import pyref
from oracle import unsaferow as U
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa
from util import assert_columns_equal

pytestmark = pytest.mark.gpu

SCH = K.example_schema()
BA = TFR_RT_BYTE_ARRAY
BA_SCH = StructType([StructField("value", BinaryType())])


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def delta(s0, s1):
    return {k: s1[k] - s0[k] for k in s0}


def frame(p):
    return pyref.frame_fast(p)


def flip(fr: bytes, pos: int, bit: int) -> bytes:
    b = bytearray(fr)
    b[pos] ^= 1 << bit
    return bytes(b)


def place(frames, rec: bytes, start: int, pad_fn) -> int:
    """append a pad record that puts the payload of `rec` at `start` mod 16 in the buffer, then `rec`; -> rec's row"""
    pos = sum(len(f) for f in frames)
    r = (start - (pos + 32 + 12)) % 16          # the pad's payload is 16 + r bytes, its frame 32 + r
    frames.append(frame(pad_fn(16 + r)))
    frames.append(rec)
    return len(frames) - 1


def check(b, used, want, what):
    info = dict(b.info)
    for k in ("error_code", "error_row", "n_rows"):
        assert info[k] == want.info[k], f"{what}: {k} {info[k]} != {want.info[k]} ({info} / {want.info})"
    assert used == want.info["consumed_bytes"], f"{what}: consumed {used} != {want.info['consumed_bytes']}"
    assert_columns_equal(b.to_host(), want.columns, None, what)


def odd_device(data: bytes):
    import torch
    buf = torch.zeros(len(data) + 1, dtype=torch.uint8, device="cuda")
    buf[1:] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    return buf, (buf.data_ptr() + 1, len(data), 1)


def sample_flips(R, positions, L, keep=4):
    """all positions of a short payload; on a long one the two stored CRCs and `keep` payload positions"""
    if L <= 1024:
        return positions
    body, crcs = positions[:-2], positions[-2:]
    return sorted(R.sample(body, min(keep, len(body)))) + crcs


# ---------------------------------------------------------------------------------------------
# synchronous decode paths
# ---------------------------------------------------------------------------------------------
def _lengths(*sets, lo=0, hi=1 << 30, ok=lambda L: True):
    return sorted({L for s in sets for L in s if lo <= L <= hi and ok(L)})


def _ex_tile_ok(L):
    return L != 0 and K.example_lengths_ok(L)         # (an empty payload is not an Example the tile takes: general path)


SYNC_PATHS = {
    # name: (record type, payload fn, lengths, flips (L, start) -> framed offsets, selector payload, stat, env general)
    "general": (0, K.example_payload,
                _lengths(K.small_lengths(), K.warp_lengths(), K.chunk_lengths(3), ok=K.example_lengths_ok),
                lambda L, s: K.warp_flips(L, s), None, "general_path_batches", True),
    "tile_4_1": (0, K.example_payload,
                 _lengths(K.small_lengths(), K.chunk_lengths(1), K.chunk_lengths(3), K.warp_lengths(),
                          [K.MAX_SLOT_PAYLOAD["tile_4_1"]], hi=K.MAX_SLOT_PAYLOAD["tile_4_1"], ok=_ex_tile_ok),
                 lambda L, s: K.chunk_flips(L, s, 1), None, "count_mode_batches", False),
    "tile_12_3": (0, K.example_payload,
                  _lengths(K.small_lengths(), K.chunk_lengths(3), K.warp_lengths(), [K.MAX_SLOT_PAYLOAD["tile_12_3"]],
                           hi=K.MAX_SLOT_PAYLOAD["tile_12_3"], ok=_ex_tile_ok),
                  lambda L, s: K.chunk_flips(L, s, 3), 2000, "count_mode_batches", False),
    "bytes_4_2": (BA, K.bytes_payload,
                  _lengths(K.small_lengths(), K.chunk_lengths(4), K.chunk_lengths(8), [K.MAX_SLOT_PAYLOAD["bytes_4_2"]],
                           hi=K.MAX_SLOT_PAYLOAD["bytes_4_2"]),
                  lambda L, s: K.chunk_flips(L, s, 4), None, "count_mode_batches", False),
    "bytes_8_4": (BA, K.bytes_payload,
                  _lengths(K.small_lengths(), K.chunk_lengths(8), K.warp_lengths(), [K.MAX_SLOT_PAYLOAD["bytes_8_4"]],
                           hi=K.MAX_SLOT_PAYLOAD["bytes_8_4"]),
                  lambda L, s: K.chunk_flips(L, s, 8), 2000, "count_mode_batches", False),
}


def _decoder(native, rt, general):
    sch = BA_SCH if rt == BA else SCH
    if not general:
        return native.Decoder(sch, rt)
    os.environ["TFR_DISABLE_FAST"] = "1"
    try:
        return native.Decoder(sch, rt)
    finally:
        del os.environ["TFR_DISABLE_FAST"]


def _on_path(name, d, stat):
    assert d[stat] == 1, (name, d)
    if stat != "general_path_batches":
        assert d["general_path_batches"] == 0 and d["large_record_batches"] == 0, (name, d)


@pytest.mark.parametrize("name", list(SYNC_PATHS))
def test_sync_decode_path(native, oracle, name):
    rt, pay, lengths, flips, selector, stat, general = SYNC_PATHS[name]
    sch = BA_SCH if rt == BA else SCH
    dec = _decoder(native, rt, general)
    R = random.Random(name)
    tail = [frame(pay(selector, seed=9))] if selector else []

    def run(data, what, expect_path):
        want = oracle.decode(data, sch, rt)
        s0 = dec.stats()
        b, used = dec.decode(data)
        check(b, used, want, what)
        b.release()
        if expect_path:
            _on_path(what, delta(s0, dec.stats()), stat)
        return want

    try:
        # clean: every length at every start offset mod 16.  A batch of 64 records or fewer teaches the decoder no sizes, so
        # every decode here is synchronous and takes the geometry of its own records
        for i, L in enumerate(lengths):
            frames = []
            for s in range(16):
                place(frames, frame(pay(L, seed=s)), s, pay)
            data = b"".join(frames + tail)
            assert len(frames) + len(tail) <= 64
            want = run(data, f"{name}: clean, L={L}", True)
            assert want.info["error_code"] == 0 and want.n_rows == len(frames) + len(tail)
            if i == len(lengths) - 1:                   # the same bytes from a device buffer at an odd address
                keep, src = odd_device(data)
                s0 = dec.stats()
                b, used = dec.decode(src)
                check(b, used, want, f"{name}: odd address")
                b.release()
                _on_path(f"{name}: odd address", delta(s0, dec.stats()), stat)
        # damaged: one flipped bit per batch, then the same batch clean
        for L in lengths:
            for s in sorted({L % 16, (7 * L + 3) % 16}):
                rec = frame(pay(L, seed=s))
                for p in sample_flips(R, flips(L, s), L):
                    frames = []
                    row = place(frames, flip(rec, p, p % 8), s, pay)
                    what = f"{name}: L={L} start={s} flip at framed byte {p}"
                    want = run(b"".join(frames + tail), what, False)
                    assert want.info["error_code"] != 0 and want.info["error_row"] == row, (what, want.info)
                frames = []
                place(frames, rec, s, pay)
                run(b"".join(frames + tail), f"{name}: L={L} start={s} clean after damage", True)
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# the packed 12 + 3 tile of a pipelined submit
# ---------------------------------------------------------------------------------------------
PACKED_BIG = [K.CHUNK * 768 + 5, K.CHUNK * 1536 + 7, 38_000]       # 12.3 KB, 24.6 KB, 38 KB


class Packed:
    def __init__(self, native, oracle):
        self.native, self.oracle = native, oracle
        R = random.Random(17)
        self.small = [K.example_payload(R.choice([L for L in range(300, 601) if K.example_lengths_ok(L)]), seed=i)
                      for i in range(96)]
        self.dec = native.Decoder(SCH)
        mix = list(self.small)
        mix[40] = K.example_payload(6000, seed=1)
        mix = b"".join(frame(p) for p in mix)
        b, used = self.dec.decode(mix)                      # learns the shapes and the largest record
        check(b, used, oracle.decode(mix, SCH), "packed: learning decode")
        b.release()
        self.submit(mix, "packed: first submit (fixed slots; learns the packed tile size)", steady=False)

    def batch(self, big_len, row, start, damage=None):
        """the small records with one record of big_len bytes at `row`, its payload at `start` mod 16 (the record in front
        of it is lengthened by up to 15 bytes); `damage`: (framed offset, bit) to flip in the big record"""
        frames = [frame(p) for p in self.small]
        pos = sum(len(f) for f in frames[:row])
        if row:
            r = (start - (pos + 12)) % 16
            prev = self.small[row - 1]
            L = len(prev) + r
            frames[row - 1] = frame(K.example_payload(L if K.example_lengths_ok(L) else L + 16, seed=row))
            pos = sum(len(f) for f in frames[:row])
        assert row == 0 or (pos + 12) % 16 == start % 16
        rec = frame(K.example_payload(big_len, seed=big_len))
        if damage:
            rec = flip(rec, *damage)
        frames[row] = rec
        return b"".join(frames), (pos + 12) % 16

    def submit(self, data, what, steady=True):
        want = self.oracle.decode(data, SCH)
        s0 = self.dec.stats()
        b = self.dec.submit(data)
        check(b, b.info["consumed_bytes"], want, what)
        b.release()
        d = delta(s0, self.dec.stats())
        if steady:
            assert d["speculative_submits"] == 1 and d["speculative_redone"] == 0, (what, d)
            assert d["general_path_batches"] == 0 and d["large_record_batches"] == 0, (what, d)
        return want

    def close(self):
        self.dec.close()


def test_packed_tile(native, oracle):
    H = Packed(native, oracle)
    R = random.Random(3)
    try:
        n = len(H.small)
        for L in PACKED_BIG:
            for row in (0, 31, 32, n - 1):
                for start in ((0,) if row == 0 else (0, 1, 8, 15)):
                    data, s = H.batch(L, row, start)
                    H.submit(data, f"packed: clean, {L} B at row {row}, start {s}")
        for L in PACKED_BIG:
            data, s = H.batch(L, 31, 5)
            for p in sample_flips(R, K.chunk_flips(L, s, 3), L, keep=8):
                bad, _ = H.batch(L, 31, 5, damage=(p, p % 8))
                what = f"packed: {L} B at row 31, start {s}, flip at framed byte {p}"
                want = H.submit(bad, what, steady=False)
                assert want.info["error_code"] != 0 and want.info["error_row"] == 31, (what, want.info)
                H.submit(data, what + ": the clean batch after it")
    finally:
        H.close()


# ---------------------------------------------------------------------------------------------
# the large-record kernel
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rt", [0, BA], ids=["large_example", "large_bytes"])
def test_large_crc(native, oracle, rt):
    sch, pay = (BA_SCH, K.bytes_payload) if rt == BA else (SCH, K.example_payload)
    ok = (lambda L: True) if rt == BA else _ex_tile_ok
    lengths = [L for L in [0] + K.large_lengths() if ok(L)]
    big = [frame(pay(65_536 + 1000 * i, seed=i)) for i in range(8)]     # keeps the batch on the large-record kernel
    dec = native.Decoder(sch, rt)
    R = random.Random(rt)

    def run(data, what, expect_path):
        want = oracle.decode(data, sch, rt)
        s0 = dec.stats()
        b, used = dec.decode(data)
        check(b, used, want, what)
        b.release()
        if expect_path:
            d = delta(s0, dec.stats())
            assert d["large_record_batches"] == 1 and d["general_path_batches"] == 0, (what, d)
        return want

    try:
        for L in lengths:
            frames = list(big[:4])
            for s in range(16):
                place(frames, frame(pay(L, seed=s)), s, pay)
            data = b"".join(frames + big[4:])
            run(data, f"large rt={rt}: clean L={L}", True)
            if L == lengths[-1]:
                keep, src = odd_device(data)
                s0 = dec.stats()
                b, used = dec.decode(src)
                check(b, used, oracle.decode(data, sch, rt), "large: odd address")
                b.release()
            for s in sorted({L % 16, (5 * L + 1) % 16}):
                rec = frame(pay(L, seed=s))
                for p in sample_flips(R, K.large_flips(L), L):
                    frames = list(big[:4])
                    row = place(frames, flip(rec, p, p % 8), s, pay)
                    what = f"large rt={rt}: L={L} start={s} flip at framed byte {p}"
                    want = run(b"".join(frames + big[4:]), what, False)
                    assert want.info["error_code"] != 0 and want.info["error_row"] == row, (what, want.info)
                frames = list(big[:4])
                place(frames, rec, s, pay)
                run(b"".join(frames + big[4:]), f"large rt={rt}: L={L} start={s} clean after damage", True)
        if rt == BA:
            # one record of 48 MiB + 3 bytes: the shift of every warp but the last has bits 22..25 set (x8pow[22..25])
            L = (48 << 20) + 3
            rec = frame(np.random.default_rng(48).integers(0, 256, L, dtype=np.uint8).tobytes())
            run(rec, "large: one 48 MiB record", True)
            for p in sample_flips(R, K.large_flips(L), L, keep=3):
                want = run(flip(rec, p, p % 8), f"large: 48 MiB record, flip at framed byte {p}", False)
                assert want.info["error_code"] != 0 and want.info["error_row"] == 0, want.info
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# schema inference and the resync scan (crc_warp)
# ---------------------------------------------------------------------------------------------
def _infer(native, data):
    inf = native.Infer(0)
    try:
        inf.update(data)
        return 0, inf.result()
    except native.TfrError as e:
        return e.code, None
    finally:
        inf.close()


def test_infer(native, oracle):
    lengths = _lengths(K.small_lengths(), K.warp_lengths(), ok=K.example_lengths_ok)
    R = random.Random(11)
    frames = []
    for L in lengths:
        for s in range(16):
            place(frames, frame(K.example_payload(L, seed=s)), s, K.example_payload)
    data = b"".join(frames)
    want = oracle.infer(data, 0)
    assert want[0] == 0
    assert _infer(native, np.frombuffer(data, np.uint8)) == want
    keep, _ = odd_device(data)
    assert _infer(native, keep[1:]) == want
    for L in lengths:
        s = (3 * L + 1) % 16
        rec = frame(K.example_payload(L, seed=s))
        for p in sample_flips(R, K.warp_flips(L, s), L):
            if p < 12:                                   # (a damaged length CRC is a framing error, not a CRC_DATA)
                continue
            fr = []
            place(fr, flip(rec, p, p % 8), s, K.example_payload)
            got = _infer(native, b"".join(fr))
            assert got == (A.TFR_E_CRC_DATA, None), (L, s, p, got)


def test_resync(native, oracle):
    import test_gpu_resync as RS
    flags = A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED | A.TFR_F_RESYNC
    lengths = _lengths(K.warp_lengths(), [13, 14, 15, 16, 17, 31, 32, 33], ok=K.example_lengths_ok)
    dec = native.Decoder(SCH, 0, 0, flags)
    R = random.Random(13)
    try:
        for L in lengths:
            frames = [frame(K.example_payload(100, seed=1))]
            frames[0] = flip(frames[0], 8 + R.randrange(4), R.randrange(8))     # a damaged length CRC in front
            for s in range(16):
                place(frames, frame(K.example_payload(L, seed=s)), s, K.example_payload)
            data = b"".join(frames)
            exp = RS.expected(oracle, data, SCH, 0, flags)
            assert RS.regions_of(exp), L
            s0 = dec.stats()
            b, used = dec.decode(data)
            assert used == exp.info["consumed_bytes"] == len(data)
            RS.check_batch(b, SCH, exp, f"resync: L={L}", rows=False)
            b.release()
            d = delta(s0, dec.stats())
            assert d["lost_regions"] == len(RS.regions_of(exp)), (L, d)
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# encoders
# ---------------------------------------------------------------------------------------------
def check_frames(got: bytes, want: bytes, what: str):
    """got == want byte for byte; otherwise name the first frame whose length CRC or data CRC is wrong"""
    if got == want:
        return
    pos, i = 0, 0
    while pos + 16 <= len(got):
        n = struct.unpack_from("<Q", got, pos)[0]
        if struct.unpack_from("<I", got, pos + 8)[0] != oracle_masked(got[pos:pos + 8]):
            raise AssertionError(f"{what}: frame {i} at {pos}: length CRC wrong")
        p = got[pos + 12:pos + 12 + n]
        if struct.unpack_from("<I", got, pos + 12 + n)[0] != oracle_masked(p):
            raise AssertionError(f"{what}: frame {i} at {pos} ({n} B payload): data CRC wrong")
        if got[pos:pos + 16 + n] != want[pos:pos + 16 + n]:
            raise AssertionError(f"{what}: frame {i} at {pos}: bytes differ from the oracle's")
        pos += 16 + n
        i += 1
    raise AssertionError(f"{what}: {len(got)} bytes, the oracle wrote {len(want)}")


def oracle_masked(b):
    from oracle import oracle
    return oracle.masked_crc32c(b)


def _example_rows(lengths, seed):
    R = random.Random(seed)
    rows = []
    for L in lengths:
        if L == 2:
            rows.append((None,))
            continue
        if L < K.MIN_EXAMPLE or not K.example_lengths_ok(L):
            continue
        v = L - K.MIN_EXAMPLE
        while v > 0 and K._example_len(v) > L:
            v -= 1
        if K._example_len(v) == L:
            rows.append((R.randbytes(v),))
    return rows


def _encode_all_ways(native, oracle, sch, rt, rows, what, general):
    cols = A.columns_from_rows(sch, rows, rt)
    want, rc, _ = oracle.encode(cols, sch, rt)
    assert rc == 0
    enc = native.Encoder(sch, rt)
    try:
        check_frames(enc.encode(cols), want, f"{what}: encode")
        data = U.unsafe_rows(sch, rows)
        enc.encode_rows(*data)
        check_frames(enc.result_host(), want, f"{what}: encode_rows")
        for k in range(3):                                  # the first submit learns, the next ones are pipelined (GUARD)
            s0 = enc.stats()
            e = enc.submit_rows(*data)
            check_frames(e.result_host(), want, f"{what}: submit_rows #{k}")
            e.release()
            d = delta(s0, enc.stats())
            assert d["general_emit"] == (1 if general else 0), (what, k, d)
            assert d["speculative_redone"] == 0, (what, k, d)
    finally:
        enc.close()


ENC_EXAMPLE_LENGTHS = _lengths([2], K.small_lengths(), K.chunk_lengths(K.ENC_WARPS), K.warp_lengths(), [6000])


def test_encode_tile(native, oracle):
    rows = _example_rows(ENC_EXAMPLE_LENGTHS, 1)
    assert len(rows) > 150
    _encode_all_ways(native, oracle, SCH, 0, rows, "encode tile", False)


def test_encode_general(native, oracle):
    rows = _example_rows(ENC_EXAMPLE_LENGTHS + [8000, 20_000, 70_000], 2)
    _encode_all_ways(native, oracle, SCH, 0, rows, "general emit (records above the slot)", True)
    rows = _example_rows(ENC_EXAMPLE_LENGTHS, 3)
    _encode_all_ways(native, oracle, SCH, TFR_RT_SEQUENCE_EXAMPLE, rows, "general emit (SequenceExample)", True)


@pytest.mark.parametrize("kind", ["enc_bytes_4_2", "enc_bytes_8_4"])
def test_encode_bytes(native, oracle, kind):
    top = K.MAX_SLOT_PAYLOAD[kind]
    C = 4 if kind == "enc_bytes_4_2" else 8
    lengths = _lengths(K.small_lengths(), K.chunk_lengths(C), K.warp_lengths(), [top], hi=top)
    R = random.Random(kind)
    rows = [(R.randbytes(L),) for L in lengths]
    _encode_all_ways(native, oracle, BA_SCH, BA, rows, kind, False)
