"""Host tests of crc_corpus: payloads of exact lengths, the length sets and flip positions of each GPU CRC-32C split, and a
model of the tile kernels' split with its shift past the xp16 table, checked against the bitwise CRC."""
import random

import crc_corpus as K
from oracle import pyref


def all_lengths():
    s = set(K.small_lengths()) | set(K.warp_lengths()) | set(K.xp16_edge_lengths()) | set(K.large_lengths())
    for C in K.TILE_CW + K.BYTES_CW + (K.ENC_WARPS,):
        s |= set(K.chunk_lengths(C))
    return sorted(s | set(K.MAX_SLOT_PAYLOAD.values()))


def test_example_payloads_have_exact_lengths_and_decode(oracle):
    lengths = [L for L in all_lengths() if K.example_lengths_ok(L)] + [133, 139, 142, 145, 16391, 16398, 16402, 16406]
    pays = [K.example_payload(L, seed=1) for L in lengths]
    assert [len(p) for p in pays] == lengths
    data = b"".join(pyref.frame(p) for p in pays)
    got = oracle.decode(data, K.example_schema())
    assert got.info["error_code"] == 0 and got.n_rows == len(lengths), got.info
    ex = pyref._cls("Example")
    want = [ex.FromString(p).features.feature["b"].bytes_list.value[0] if len(p) >= K.MIN_EXAMPLE else None for p in pays]
    assert [r[0] for r in got.rows()] == want


def test_every_example_length_from_the_smallest_one():
    assert [L for L in range(20_000) if not K.example_lengths_ok(L)] == [1] + list(range(3, K.MIN_EXAMPLE)) + [130, 16387]
    for L in range(20_000):
        if K.example_lengths_ok(L):
            assert len(K.example_payload(L)) == L, L


def test_bytes_payloads_have_exact_lengths():
    for L in all_lengths():
        assert len(K.bytes_payload(L, seed=2)) == L


def test_bitwise_crc_agrees_with_the_oracle_on_every_length(oracle):
    R = random.Random(3)
    for L in all_lengths():
        p = R.randbytes(L)
        assert pyref.crc32c(p) == oracle.crc32c(p), L
        assert pyref.masked_crc32c(p) == oracle.masked_crc32c(p), L


def test_length_sets_hold_their_boundaries():
    for C in (3, 4, 8):
        s = set(K.chunk_lengths(C))
        for k in (C - 1, C, C + 1, 2 * C - 1, 2 * C, 2 * C + 1):
            assert {16 * k, 16 * k + 1, 16 * k + 15} <= s, (C, k)
    w = set(K.warp_lengths())
    assert {128, 129, 131, 132, 133, 128 * 32, 128 * 33 + 5} <= w
    assert set(range(0, 161)) == set(K.small_lengths())
    x = set(K.xp16_edge_lengths())
    assert {16 * 511, 16 * 767, 16 * 767 + 15, 16 * 1535, 16 * 1536 + 15} <= x
    lg = set(K.large_lengths())
    assert set(range(1, 17)) <= lg and {23, 25, 65535, 65537} <= lg
    # where the 12 + 3 tile's warps 0 and 1 first shift by 512 chunks or more
    assert K.first_xp16_overflow(3) == 767
    assert min(k for k in range(1, 4000) if k - 2 * k // 3 >= K.XP16) == 1534
    # the other xp16 users never get there with the payloads their fixed slots take: the ByteArray kernels (C = 4, 8) and the
    # Example encode tile (8 warps), whose slots stop near 7 KiB
    for C, path in ((4, "bytes_4_2"), (8, "bytes_8_4"), (8, "enc_bytes_8_4")):
        assert K.CHUNK * K.first_xp16_overflow(C) > K.MAX_SLOT_PAYLOAD[path], (C, path)
    assert K.CHUNK * K.first_xp16_overflow(K.ENC_WARPS) > 8192


def test_flip_positions():
    L, start = 1000, 5
    pos = K.chunk_flips(L, start, 3)
    hn = 11                                  # (-5) mod 16
    k = (L - hn) // 16                       # 61 chunks, warps [0, 20) [20, 40) [40, 61)
    want = {12, 12 + hn - 1, 12 + hn, 12 + hn + 16 * 20 - 1, 12 + hn + 16 * 20, 12 + hn + 16 * 40 - 1, 12 + hn + 16 * 40,
            12 + hn + 16 * k - 1, 12 + hn + 16 * k, 12 + L - 1, 12 + L + 2, 9}
    assert set(pos) == want
    for L in all_lengths():
        for start in range(16):
            for C in (1, 3, 4, 8):
                ps = K.chunk_flips(L, start, C)
                assert all(0 <= p < L + 16 for p in ps) and len(set(ps)) == len(ps)
        ps = K.warp_flips(L, 3)
        assert all(0 <= p < L + 16 for p in ps)
    assert K.large_flips(3) == [12, 13, 14, 17, 9]       # warps 2, 5, 7 own one byte each, the others none


def test_tile_split_model_matches_the_bitwise_crc(oracle):
    """the kernels' split (head byte-wise, K chunks over C warps joined by chunk_shift, tail byte-wise) is the CRC for every
    start offset, at the chunk counts around xp16's reach and far past it (16,383 chunks, more than any tile holds)"""
    R = random.Random(4)
    for C in (1, 3, 4, 8):
        for L in K.chunk_lengths(C) + K.small_lengths()[::7]:
            p = R.randbytes(L)
            for start in range(16):
                assert K.tile_crc(p, start, C) == oracle.crc32c(p), (C, L, start)
    for L in K.xp16_edge_lengths() + [100_000, 200_000, 16 * 16383 + 15]:
        p = R.randbytes(L)
        for start in (0, 1, 15):
            assert K.tile_crc(p, start, 3) == oracle.crc32c(p), (L, start)
    # the table alone runs out at K = 767 chunks, where warp 0 first shifts by 512
    p = R.randbytes(16 * 767)
    assert K.tile_crc(p, 0, 3, extended=False) is None
    assert K.tile_crc(p[:16 * 766], 0, 3, extended=False) == oracle.crc32c(p[:16 * 766])


def test_chunk_shift_is_the_power_of_x():
    for m in [0, 1, 511, 512, 513, 767, 1023, 1024, 1535, 4096, 16383]:
        assert K.chunk_shift(m) == K.xpow_bytes(16 * m), m
    assert K.chunk_shift(512, extended=False) is None
