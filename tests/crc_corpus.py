"""Payloads of exact lengths, and the lengths and bit-flip positions at which the GPU's CRC-32C routines change how they
split a payload (csrc/tile.cuh, bytes_tile.cuh, encode_tile.cuh, common.cuh crc_warp, large.cuh large_crc).

Every set here is computed from the split parameters of the routine it is for -- the number of CRC warps C, 16-byte
chunks, 4-byte words over 32 lanes, the 512 entries of the xp16 shift table, the 8 warps of the large-record kernel --
so that a change of those parameters moves the tested boundaries with it."""
from __future__ import annotations

import random

from oracle import pyref
from spark_tfrecord_b200.sqltypes import BinaryType, StructField, StructType

CHUNK = 16            # the tile kernels fold 16-byte chunks
WORD = 4              # crc_warp: lane l folds the words l, l + 32, ...
LANES = 32
XP16 = 512            # entries of the xp16 table: x^(8*16*m) for m < 512
LARGE_WARPS = 8       # large_crc: one byte range per warp
TILE_CW = (1, 3)      # CRC warps of the 4 + 1 and 12 + 3 decode tiles
BYTES_CW = (4, 8)     # CRC warps of the ByteArray kernels <4,2> and <8,4> (decode and encode)
ENC_WARPS = 8         # the Example encode tile: every warp folds a share of each record

# The largest payload each fixed-slot kernel accepts on an H100 (227 KiB opt-in shared memory per CTA, 228 KiB per SM with
# 1 KiB reserved per CTA), for a synchronous decode or encode of the one-BinaryType-field schema below.  A slot is an odd
# number of 16-byte units: decode align16(L + 16 + 15 + 32), ByteArray encode align16(L + 78); 32 slots per tile.
#   decode 4 + 1 tile      8 tiles per SM: 32 * 688 B slots                                      L <= 625
#   decode 12 + 3 tile     one tile of 32 * 7088 B slots                                         L <= 7025
#   ByteArray decode <4,2> 10 tiles per SM: 32 * 528 B slots                                     L <= 465
#   ByteArray decode <8,4> 32 * 7088 B slots                                                     L <= 7025
#   ByteArray encode <4,2> 32 * 528 B slots                                                      L <= 450
#   ByteArray encode <8,4> 32 * 7088 B slots                                                     L <= 7010
MAX_SLOT_PAYLOAD = {"tile_4_1": 625, "tile_12_3": 7025, "bytes_4_2": 465, "bytes_8_4": 7025,
                    "enc_bytes_4_2": 450, "enc_bytes_8_4": 7010}

MIN_EXAMPLE = 13      # 0A 0B | 0A 09 | 0A 01 'b' 12 04 | 0A 02 | 0A 00: one feature holding an empty bytes value


def example_schema() -> StructType:
    return StructType([StructField("b", BinaryType())])


def _vsize(v: int) -> int:
    return len(pyref.varint(v))


def _example_len(v: int) -> int:
    """payload bytes of the one-feature Example whose bytes value has v bytes"""
    bl = 1 + _vsize(v) + v                 # BytesList { value = 1 }
    f = 1 + _vsize(bl) + bl                # Feature { bytes_list = 1 }
    e = 3 + 1 + _vsize(f) + f              # map entry { key = 1 ("b"), value = 2 }
    g = 1 + _vsize(e) + e                  # Features { feature = 1 }
    return 1 + _vsize(g) + g               # Example { features = 1 }


def _example(value: bytes, pad_width: int) -> bytes:
    feats = {"b": pyref.bytes_feature(value)}
    if pad_width:                          # an int64 feature the schema does not read, its value a varint of pad_width bytes
        feats["p"] = pyref.int64_feature(1 << (7 * (pad_width - 1)) if pad_width < 10 else -1)
    return pyref.example(feats).SerializeToString()


def example_payload(L: int, seed: int = 0) -> bytes:
    """an Example payload of exactly L bytes: the empty payload (L = 0), an Example with no features (0A 00, L = 2), or the
    BinaryType feature "b" (L >= MIN_EXAMPLE).  The payload grows by one byte per value byte except where one of its five
    varints gains a byte, which skips a length (130, 133, 139, 142, 145, 16387, ...); those lengths take a second feature "p"
    that the schema does not read, its int64 value sized (1 to 10 varint bytes) to close the gap.  No canonical Example has
    a length example_lengths_ok rejects."""
    if L == 0:
        return b""
    if L == 2:
        return b"\x0a\x00"
    assert example_lengths_ok(L), L
    v = max(0, L - MIN_EXAMPLE)
    while v > 0 and _example_len(v) > L:
        v -= 1
    value = random.Random(seed * 1_000_003 + L).randbytes(L)
    if _example_len(v) == L:
        return _example(value[:v], 0)
    for w in range(1, 11):
        extra = len(_example(b"", w)) - MIN_EXAMPLE
        for u in range(max(0, v - extra - 8), v + 1):
            p = _example(value[:u], w)
            if len(p) == L:
                return p
    raise ValueError(f"no Example payload of {L} bytes")


def bytes_payload(L: int, seed: int = 0) -> bytes:
    return random.Random(seed * 1_000_003 + L).randbytes(L)


def example_lengths_ok(L: int) -> bool:
    """whether some canonical Example payload has L bytes: 0, 2, and every L >= MIN_EXAMPLE except those the outer length
    varint jumps over (130, 16387, ...: an Example with Features of 127 bytes has 129, of 128 bytes 131)"""
    if L in (0, 2):
        return True
    return L >= MIN_EXAMPLE and any(1 + _vsize(g) + g == L for g in (L - 2, L - 3, L - 4, L - 5))


# ---------------------------------------------------------------------------------------------
# length sets
# ---------------------------------------------------------------------------------------------
def small_lengths() -> list:
    """every length of a head, a few chunks and a tail, for every routine"""
    return list(range(0, 161))


def chunk_counts(C: int) -> list:
    """chunk counts around where C warps' ranges [K c / C, K (c + 1) / C) go from empty to one and two chunks"""
    return sorted({k for k in (C - 1, C, C + 1, 2 * C - 1, 2 * C, 2 * C + 1) if k >= 0})


def chunk_lengths(C: int) -> list:
    """payloads of K whole chunks, one byte of tail, and a full 15-byte tail"""
    return sorted({CHUNK * k + t for k in chunk_counts(C) for t in (0, 1, 15)})


def warp_lengths() -> list:
    """crc_warp: m rows of 32 words, then 0, 1, 3 tail bytes (n & 3) and a 33rd word"""
    row = LANES * WORD
    return sorted({row * m + t for m in (1, 2, 31, 32, 33) for t in (0, 1, 3, 4, 5)})


XP16_EDGE_CHUNKS = (XP16 - 1, XP16, 766, 767, 768, 1534, 1535, 1536)


def xp16_edge_lengths() -> list:
    """payloads of K chunks around the reach of xp16: the 12 + 3 tile's warp 0 shifts by K - floor(K / 3), which is 512
    from K = 767 on; warp 1 by K - floor(2K / 3), 512 from K = 1534 on"""
    return sorted({CHUNK * k + t for k in XP16_EDGE_CHUNKS for t in (0, 15)})


def large_lengths() -> list:
    """large_crc: 1..16 bytes (some of the 8 warps get empty ranges), and 8m +- 1 (uneven ranges)"""
    return sorted(set(range(1, 17)) | {LARGE_WARPS * m + d for m in (3, 16, 128, 4096, 8192) for d in (-1, 1)})


def first_xp16_overflow(C: int) -> int:
    """the smallest chunk count at which some warp of a C-warp split shifts by XP16 chunks or more"""
    K = 1
    while max(K - K * (cw + 1) // C for cw in range(C)) < XP16:
        K += 1
    return K


# ---------------------------------------------------------------------------------------------
# bit-flip positions
# ---------------------------------------------------------------------------------------------
def _framed(positions, L):
    """payload byte indices -> framed record offsets (the payload starts 12 bytes in), plus one bit of each stored CRC"""
    out = sorted({12 + i for i in positions if 0 <= i < L})
    return out + [12 + L + 2, 8 + 1]            # a bit of the stored data CRC, a bit of the stored length CRC


def chunk_flips(L: int, start: int, C: int) -> list:
    """framed-record offsets to damage for a C-warp tile split of an L-byte payload starting at `start` mod 16: the first
    byte, the last byte before the first 16-byte boundary, the first and last byte of each warp's chunk range, the first
    tail byte, the last byte, and the two stored CRCs"""
    hn = min(L, (-start) % CHUNK)
    K = (L - hn) // CHUNK
    pos = [0, hn - 1, hn + CHUNK * K, L - 1]
    for cw in range(C):
        k0, k1 = K * cw // C, K * (cw + 1) // C
        if k1 > k0:
            pos += [hn + CHUNK * k0, hn + CHUNK * k1 - 1]
    return _framed(pos, L)


def warp_flips(L: int, start: int) -> list:
    """crc_warp over an L-byte payload at `start` mod 4: the first byte, the end of the first aligned word, the first and
    last byte of the second 128-byte row, the first tail byte (n & 3) and the last byte, and the two stored CRCs"""
    a = (-start) % WORD
    W = L // WORD
    pos = [0, a - 1, LANES * WORD, 2 * LANES * WORD - 1, WORD * W, L - 1]
    return _framed(pos, L)


def large_flips(L: int) -> list:
    """large_crc: the first and last byte of every warp's byte range, and the two stored CRCs"""
    pos = []
    for w in range(LARGE_WARPS):
        lo, hi = L * w // LARGE_WARPS, L * (w + 1) // LARGE_WARPS
        if hi > lo:
            pos += [lo, hi - 1]
    return _framed(pos, L)


# ---------------------------------------------------------------------------------------------
# a model of the tile kernels' split (csrc/tile.cuh, crc_chunks + chunk_shift), for the host tests
# ---------------------------------------------------------------------------------------------
POLY = 0x82F63B78


def _table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ (POLY if c & 1 else 0)
        t.append(c)
    return t


T0 = _table()


def crc_raw(c: int, data: bytes) -> int:
    for b in data:
        c = (c >> 8) ^ T0[(c ^ b) & 0xFF]
    return c


def gf2_mulmod(a: int, b: int) -> int:
    """GF(2) product mod P in the reflected bit order (bit 31 = x^0), as common.cuh's"""
    p = 0
    for i in range(31, -1, -1):
        if (a >> i) & 1:
            p ^= b
        b = (b >> 1) ^ (POLY if b & 1 else 0)
    return p


def xpow_bytes(n: int) -> int:
    """x^(8 n) mod P"""
    r, base = 0x80000000, 0x80000000
    for _ in range(8):
        base = (base >> 1) ^ (POLY if base & 1 else 0)
    while n:
        if n & 1:
            r = gf2_mulmod(r, base)
        base = gf2_mulmod(base, base)
        n >>= 1
    return r


XP16_TABLE = [xpow_bytes(CHUNK * m) for m in range(XP16)]


def chunk_shift(m: int, extended: bool = True):
    """the kernel's factor x^(8*16*m): xp16[m] below 512; beyond, xp16[511] once per 511 chunks times xp16 of the rest.
    None where only the table is used and m is past it."""
    if m < XP16:
        return XP16_TABLE[m]
    if not extended:
        return None
    f, m = XP16_TABLE[XP16 - 1], m - (XP16 - 1)
    while m:
        s = min(m, XP16 - 1)
        f = gf2_mulmod(f, XP16_TABLE[s])
        m -= s
    return f


def tile_crc(payload: bytes, start: int, C: int, extended: bool = True):
    """CRC-32C of the payload as a C-warp tile computes it (head byte-wise, K chunks split over the warps and joined by
    shifts, tail byte-wise); None if a shift leaves the table (extended=False)"""
    L = len(payload)
    hn = min(L, (-start) % CHUNK)
    K = (L - hn) // CHUNK
    acc = 0
    for cw in range(C):
        k0, k1 = K * cw // C, K * (cw + 1) // C
        c = crc_raw(0xFFFFFFFF, payload[:hn]) if cw == 0 else 0
        c = crc_raw(c, payload[hn + CHUNK * k0:hn + CHUNK * k1])
        if K - k1 and c:
            s = chunk_shift(K - k1, extended)
            if s is None:
                return None
            c = gf2_mulmod(s, c)
        acc ^= c
    return crc_raw(acc, payload[hn + CHUNK * K:]) ^ 0xFFFFFFFF
