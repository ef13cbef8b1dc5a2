"""Seeded wire-format rewriter for the decode parity tests.  TEST INFRASTRUCTURE ONLY.

A record of a random schema is serialised the way the reference writer serialises it (`canonical`: map entries in schema
order, key then value, packed numeric lists, minimal varints, M/TFRecordSerializer.scala:20-60) and then rewritten into
another wire form that protobuf-java parses to the same message (class A, `rewrite`), into a record whose row fails with
a known status (class B, `error_record`), or damaged byte-wise (class C, `mutate`).  Every payload is built from the
`oracle/pyref.py` helpers and framed with a valid CRC, so it reaches the parsers instead of stopping at the CRC check.

Class A names (`A_CLASSES`) and what they rewrite:
  order        map entries reversed, shuffled, or rotated so that ownership `i mod W` shifts for W = 12 and W = 4
  extra        a feature the schema does not have, anywhere: every kind and kind-not-set; keys of 0, 1, 12, 13 and 300
               bytes, a schema key +- one byte, multibyte UTF-8, a key with a schema key's FNV-1a hash, a key in a schema
               key's hash-table slot
  null_present a NullType schema field present with a value of any kind
  multibyte    a feature of 128+ bytes (real multibyte lengths at every level)
  many_entries more map entries than the tile kernel's entry table has rows (one per schema field)
  overlong     one length or tag as an overlong varint, at elen / klen / vlen / llen / plen / blen / a tag
  unpacked     numeric lists unpacked, mixed packed and unpacked, or in packed segments (empty ones included)
  merge        a Feature given twice with its list split, a oneof decoy of another kind first, the same kind twice,
               `features` (or context / feature_lists) split across two fields, an earlier decoy entry for the same key
               at an entry distance of 0 or not 0 mod W
  entry_inner  value before key; key twice, decoy first
  unknown      unknown fields of all five wire types (nested groups included) at the Example, Features, entry, Feature and
               list levels, and known field numbers with the wrong wire type
  seq          SequenceExample: feature_lists before context, an empty one omitted, each split in two, a FeatureList given
               twice in an entry (its steps concatenate), unknown fields in FeatureList and FeatureLists
  size         a payload over 64 KiB whose schema entries sit past 64 KiB, a FeatureList over 4 KiB, a non-canonical
               cell group over 2 KiB

The first five classes keep the writer's canonical shape (tile.cuh: payload / Features / Feature / List): a decoder's
fast path must take them.  Every rewrite returns a tag naming what was done, for failure messages.
"""
from __future__ import annotations

import random
import struct
from functools import lru_cache
from typing import List, Optional, Tuple

import numpy as np

from oracle import pyref
from oracle.pyref import ld, tag, varint
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import (ArrayType, BinaryType, DoubleType, FloatType, IntegerType, LongType, NullType,
                                          StringType, StructField, StructType, TFR_RT_SEQUENCE_EXAMPLE)

A_CLASSES = ["order", "extra", "null_present", "multibyte", "many_entries", "overlong", "unpacked", "merge", "entry_inner",
             "unknown", "seq", "size"]
CANONICAL_CLASSES = {"order", "extra", "null_present", "multibyte", "many_entries"}
B_CLASSES = ["kind_mismatch", "kind_not_set", "empty_scalar", "null_in_nonnull", "bad_nesting", "malformed", "groups_24",
             "groups_25"]
MAL_SHAPES = {      # appended to a valid payload at its top level (each is one `mal_*` shape of tests/cases.py)
    "mal_truncated_len": bytes([0x0A, 0x05, 0x0A]),
    "mal_varint_too_long": ld(1, pyref.map_entry(b"k", ld(3, ld(1, bytes([0x80] * 10 + [0x01]))))),
    "mal_truncated_varint": ld(1, pyref.map_entry(b"k", ld(3, ld(1, bytes([0x80]))))),
    "mal_packed_float_ragged": ld(1, pyref.map_entry(b"f", ld(2, ld(1, b"abcde")))),
    "mal_fixed32_truncated": ld(1, pyref.map_entry(b"f", ld(2, tag(1, 5) + b"abc"))),
    "mal_tag_zero": ld(1, bytes([0x00])),
    "mal_field_number_zero": ld(1, pyref.map_entry(b"k", bytes([0x02, 0x00]))),
    "mal_wiretype_6": ld(1, pyref.map_entry(b"k", bytes([0x0E]))),
    "mal_wiretype_7_toplevel": bytes([0x0F]),
    "mal_stray_end_group": ld(1, tag(3, 4)),
    "mal_unterminated_group": tag(5, 3) + tag(6, 0) + varint(1),
    "mal_mismatched_end_group": tag(5, 3) + tag(6, 4),
    "mal_invalid_utf8_key": ld(1, pyref.map_entry(b"\xff\xfe", ld(3, ld(1, varint(1))))),
    "mal_invalid_utf8_key_surrogate": ld(1, pyref.map_entry(b"\xed\xa0\x80", ld(3, ld(1, varint(1))))),
    "mal_invalid_utf8_key_overlong": ld(1, pyref.map_entry(b"\xc0\x80", ld(3, ld(1, varint(1))))),
    "mal_deep_in_unused_feature": ld(1, pyref.map_entry(b"unused", ld(1, ld(1, b"abc")[:-1]))),
    "mal_negative_length": ld(1, bytes([0x0A, 0xFF, 0xFF, 0xFF, 0xFF, 0x0F])),
    "mal_bytes_elem_overrun": ld(1, pyref.map_entry(b"b", ld(1, bytes([0x0A, 0x05, 0x61])))),
    "mal_fixed64_truncated": ld(1, tag(4, 1) + b"1234567"),
}

K_BYTES, K_FLOAT, K_INT64 = 1, 2, 3


# --------------------------------------------------------------------------------------------
# wire helpers
# --------------------------------------------------------------------------------------------
def ov(v: int, pad: int = 1) -> bytes:
    """`v` as a non-minimal varint with `pad` extra bytes (protobuf accepts up to ten bytes)"""
    b = bytearray(varint(v))
    b[-1] |= 0x80
    return bytes(b) + bytes([0x80] * (pad - 1)) + b"\x00"


def ld_ov(field: int, payload: bytes, pad: int = 1) -> bytes:
    """length-delimited field whose length is an overlong varint"""
    return tag(field, 2) + ov(len(payload), pad) + payload


def fnv1a(b: bytes) -> int:
    h = 2166136261
    for c in b:
        h = ((h ^ c) * 16777619) & 0xFFFFFFFF
    return h


def ht_mask(n_fields: int) -> int:
    """mask of the decoder's key hash table (api.cu: the smallest power of two >= 2 * fields + 2)"""
    hsz = 2
    while hsz < 2 * n_fields + 2:
        hsz <<= 1
    return hsz - 1


@lru_cache(maxsize=None)
def fnv_collision() -> Tuple[bytes, bytes]:
    """two different 8-byte lowercase ASCII keys with the same FNV-1a hash (a birthday search over 2^17 keys)"""
    rng = np.random.default_rng(20261015)
    for _ in range(64):
        keys = rng.integers(ord("a"), ord("z") + 1, (1 << 17, 8), dtype=np.uint8)
        h = np.full(len(keys), 2166136261, np.uint64)
        for i in range(8):
            h = ((h ^ keys[:, i]) * np.uint64(16777619)) & np.uint64(0xFFFFFFFF)
        order = np.argsort(h, kind="stable")
        hs = h[order]
        dup = np.nonzero(hs[1:] == hs[:-1])[0]
        for d in dup:
            a, b = keys[order[d]].tobytes(), keys[order[d + 1]].tobytes()
            if a != b:
                assert fnv1a(a) == fnv1a(b)
                return a, b
    raise AssertionError("no FNV-1a collision found")


# --------------------------------------------------------------------------------------------
# schemas and rows
# --------------------------------------------------------------------------------------------
LEAVES = [("i", IntegerType), ("l", LongType), ("f", FloatType), ("d", DoubleType), ("s", StringType), ("b", BinaryType)]


def _leaf(r, kind, short):
    if kind == "i":
        return int(r.integers(-2**31, 2**31))
    if kind == "l":
        return int(r.integers(-2**63, 2**63 - 1)) if r.random() < 0.5 else int(r.integers(-100, 100))
    if kind in ("f", "d"):
        return float(np.float32(r.standard_normal()))
    n = int(r.integers(0, 6 if short else 24))
    if kind == "s":
        return "".join(chr(int(c)) for c in r.choice([0x41, 0x7A, 0xE9, 0x4E2D, 0x1F600, 0x20], n))
    return r.integers(0, 256, n, dtype=np.uint8).tobytes()


BAD_UTF8 = [b"\xff", b"\xc3", b"\xe2\x82", b"\xed\xa0\x80", b"\xf0\x9f\x98", b"\xc0\xaf", b"ok\x80ok"]


def make_schema(seed: int, width: int, record_type: int = 0, big: bool = False, uniform: bool = False,
                bad_utf8: bool = False, flist_numeric: bool = False, with_2d: bool = False):
    """-> (StructType, row generator).  `width` fields of every leaf type, scalars and lists (and FeatureLists for a
    SequenceExample), NullType and non-nullable fields, names of 12 and 13 bytes, and one name that shares its FNV-1a
    hash with another key (`fnv_collision`).  Field 0 is a non-nullable scalar long.  `uniform`: every list has a
    fixed length and no nulls (the uniform-shape mode); otherwise lists are ragged and nullable.  `big`: a binary field
    of ~2 KiB per row makes records large.  `bad_utf8`: a ragged string column with malformed UTF-8 in some rows.
    `flist_numeric`: FeatureList columns hold numbers only.  `with_2d` (Example): one more column of type array<array<>>,
    absent from every row (an Example can only feed it a Feature, which is BAD_NESTING: error_record)."""
    rng = np.random.default_rng(seed)
    fields, gens = [], []
    coll = fnv_collision()[0].decode()
    seq = record_type == TFR_RT_SEQUENCE_EXAMPLE

    def name(j, kind):
        nm = f"c{j}_{kind}"
        if j % 7 == 3:
            nm = nm.ljust(12, "x")
        elif j % 7 == 4:
            nm = nm.ljust(13, "y")
        return nm

    for j in range(width):
        kind, dt = LEAVES[int(rng.integers(0, len(LEAVES)))]
        nm = name(j, kind)
        if j == width // 2 and width > 1:
            nm = coll
        if j == 0:
            fields.append(StructField(nm, LongType(), False))
            gens.append(lambda r: _leaf(r, "l", True))
            continue
        if width > 2 and j == 1 and big:
            L = int(rng.integers(1800, 2400))
            fields.append(StructField(nm, BinaryType(), False))
            gens.append(lambda r, L=L, u=uniform: r.integers(0, 256, L if u else int(r.integers(L - 300, L + 300)), dtype=np.uint8).tobytes())
            continue
        if bad_utf8 and j == 2 and width > 2:
            fields.append(StructField(nm, ArrayType(StringType()), True))

            def gen_bad(r):
                vals = [_leaf(r, "s", True) for _ in range(int(r.integers(0, 4)))]
                if vals and r.random() < 0.1:
                    vals[0] = BAD_UTF8[int(r.integers(0, len(BAD_UTF8)))]
                return vals
            gens.append(gen_bad)
            continue
        u = rng.random()
        if j % 11 == 7:
            fields.append(StructField(nm, NullType(), True))
            gens.append(lambda r: None)
        elif seq and u < 0.3:
            if flist_numeric and kind in "sb":
                kind, dt = "f", FloatType
            fields.append(StructField(nm + "aa", ArrayType(ArrayType(dt())), True))
            L = int(rng.integers(0, 3))

            def gen2(r, kind=kind, u=uniform, L=L):
                if not u and r.random() < 0.15:
                    return None
                return [[_leaf(r, kind, True) for _ in range(L if u else int(r.integers(0, 4)))]
                        for _ in range(2 if u else int(r.integers(0, 5)))]
            gens.append(gen2)
        elif u < 0.6 and not (uniform and kind in "sb"):
            fixed = int(rng.integers(1, 4))
            nullable = not uniform and rng.random() < 0.6
            fields.append(StructField(nm + "a", ArrayType(dt()), nullable))

            def gen1(r, kind=kind, u=uniform, fixed=fixed, nullable=nullable):
                if nullable and r.random() < 0.15:
                    return None
                return [_leaf(r, kind, True) for _ in range(fixed if u else int(r.integers(0, 5)))]
            gens.append(gen1)
        else:
            nullable = not uniform and rng.random() < 0.6
            if uniform and kind in "sb":
                kind, dt = "l", LongType
            fields.append(StructField(nm, dt(), nullable))

            def gen0(r, kind=kind, nullable=nullable):
                if nullable and r.random() < 0.15:
                    return None
                return _leaf(r, kind, True)
            gens.append(gen0)
    if seq and width > 2 and not any(isinstance(f.dataType, ArrayType) and isinstance(f.dataType.elementType, ArrayType)
                                     for f in fields):
        kind, dt = LEAVES[int(rng.integers(0, 4))]
        fields[-1] = StructField(fields[-1].name + "aa", ArrayType(ArrayType(dt())), True)
        gens[-1] = lambda r, kind=kind: [[_leaf(r, kind, True)] for _ in range(2)]
    if with_2d and not seq:
        fields.append(StructField(f"c{width}_2d", ArrayType(ArrayType(LongType())), True))
        gens.append(lambda r: None)
    sch = StructType(fields)

    def gen_row(r):
        return tuple(g(r) for g in gens)
    return sch, gen_row


# --------------------------------------------------------------------------------------------
# the writer's canonical form
# --------------------------------------------------------------------------------------------
def _leaf_type(dt):
    while isinstance(dt, ArrayType):
        dt = dt.elementType
    return dt


def kind_of(dt) -> int:
    et = _leaf_type(dt)
    if isinstance(et, (IntegerType, LongType)):
        return K_INT64
    if isinstance(et, (FloatType, DoubleType)):
        return K_FLOAT
    return K_BYTES


def elems_of(kind: int, vals) -> List[bytes]:
    if kind == K_INT64:
        return [varint(int(v)) for v in vals]
    if kind == K_FLOAT:
        return [struct.pack("<f", np.float32(v)) for v in vals]
    return [v.encode("utf-8") if isinstance(v, str) else bytes(v) for v in vals]


def list_body(kind: int, elems: List[bytes]) -> bytes:
    if kind == K_BYTES:
        return b"".join(ld(1, e) for e in elems)
    return ld(1, b"".join(elems)) if elems else b""


def feature(kind: int, elems: List[bytes]) -> bytes:
    return ld(kind, list_body(kind, elems))


def entry(key: bytes, value: bytes) -> bytes:
    return ld(1, ld(1, key) + ld(2, value))


class Field:
    """one present schema field of a record: its key, its Feature (or the steps of its FeatureList)"""

    def __init__(self, idx, key, kind, elems=None, steps=None):
        self.idx, self.key, self.kind, self.elems, self.steps = idx, key, kind, elems, steps

    @property
    def is_flist(self):
        return self.steps is not None

    def value(self) -> bytes:
        if self.is_flist:
            return b"".join(ld(1, feature(self.kind, s)) for s in self.steps)
        return feature(self.kind, self.elems)


def present_fields(schema: StructType, row) -> List[Field]:
    out = []
    for i, (f, v) in enumerate(zip(schema.fields, row)):
        if v is None or isinstance(f.dataType, NullType):
            continue
        k = kind_of(f.dataType)
        key = f.name.encode("utf-8")
        dt = f.dataType
        if isinstance(dt, ArrayType) and isinstance(dt.elementType, ArrayType):
            out.append(Field(i, key, k, steps=[elems_of(k, s) for s in v]))
        elif isinstance(dt, ArrayType):
            out.append(Field(i, key, k, elems=elems_of(k, v)))
        else:
            out.append(Field(i, key, k, elems=elems_of(k, [v])))
    return out


def assemble(record_type: int, ctx: List[bytes], fls: List[bytes]) -> bytes:
    if record_type == TFR_RT_SEQUENCE_EXAMPLE:
        return ld(1, b"".join(ctx)) + ld(2, b"".join(fls))
    return ld(1, b"".join(ctx))


def canonical(schema: StructType, row, record_type: int = 0) -> bytes:
    """the payload the reference writer produces for `row`"""
    fs = present_fields(schema, row)
    return assemble(record_type, [entry(f.key, f.value()) for f in fs if not f.is_flist],
                    [entry(f.key, f.value()) for f in fs if f.is_flist])


def source_columns(schema: StructType, rows, record_type: int = 0) -> List[A.HostColumn]:
    """the columns a decoder must produce for `rows` (a NullType column: all null, no values)"""
    cols = A.columns_from_rows(schema, rows, record_type)
    for i, c in enumerate(cols):
        if c.elem_type == A.TFR_T_NULL:
            cols[i] = A.HostColumn(c.elem_type, c.depth, c.n_rows, c.validity, c.offsets, c.values[:0])
    return cols


def frame(payloads) -> bytes:
    return b"".join(pyref.frame_fast(p) for p in payloads)


# --------------------------------------------------------------------------------------------
# class A: equivalent rewrites
# --------------------------------------------------------------------------------------------
def _unknown(R: random.Random, depth: int = 0, wt: Optional[int] = None, fno: Optional[int] = None) -> bytes:
    """one unknown field: varint, fixed64, length-delimited, group (with nested unknown fields) or fixed32"""
    wt = R.choice([0, 1, 2, 3, 5]) if wt is None else wt
    fno = fno if fno is not None else R.choice([4, 5, 9, 15, 16, 100, 2047, 2048, (1 << 29) - 1])
    if wt == 0:
        return tag(fno, 0) + varint(R.choice([0, 1, 300, 2**63, 2**64 - 1]))
    if wt == 1:
        return tag(fno, 1) + bytes(R.randrange(256) for _ in range(8))
    if wt == 2:
        return ld(fno, bytes(R.randrange(256) for _ in range(R.choice([0, 1, 5, 130]))))
    if wt == 5:
        return tag(fno, 5) + bytes(R.randrange(256) for _ in range(4))
    inner = b"".join(_unknown(R, depth + 1, R.choice([0, 1, 2, 5] + ([3] if depth < 3 else []))) for _ in range(R.randrange(3)))
    return tag(fno, 3) + inner + tag(fno, 4)


def _unknowns(R, k=None) -> bytes:
    return b"".join(_unknown(R) for _ in range(R.randrange(1, 3) if k is None else k))


def _extra_key(R: random.Random, schema: StructType, variant: str) -> bytes:
    names = {f.name.encode("utf-8") for f in schema.fields}
    base = R.choice(sorted(names))
    for attempt in range(50000):
        if variant.startswith("len"):
            n = int(variant[3:])
            k = bytes(R.choice(b"abcdefghijklmnopqrstuvwxyz_0123456789") for _ in range(n))
        elif variant == "plus_byte":
            k = base + R.choice([b"x", b"_", b"0"])
        elif variant == "minus_byte":
            k = base[:-1]
        elif variant == "utf8":
            k = R.choice(["ключ", "キー😀", "é", "中文字段名", "😀😀😀x"]).encode("utf-8") + str(attempt).encode() * (attempt > 0)
        elif variant == "fnv":
            a, b = fnv_collision()
            k = b if a in names else a
        elif variant == "slot":
            m = ht_mask(len(schema.fields))
            want = fnv1a(base) & m
            k = base + b"_%d" % R.randrange(1 << 20)
            if fnv1a(k) & m != want or fnv1a(k) == fnv1a(base):
                continue
        else:
            raise ValueError(variant)
        if k not in names:
            return k
        base = R.choice(sorted(names))
    raise AssertionError(f"no extra key for {variant}")


EXTRA_KEYS = ["len0", "len1", "len12", "len13", "len300", "plus_byte", "minus_byte", "utf8", "fnv", "slot"]


def _any_feature(R: random.Random, allow_unset=True) -> bytes:
    k = R.choice([K_BYTES, K_FLOAT, K_INT64] + ([0] if allow_unset else []))
    if k == 0:
        return b""                                        # kind not set: 12 00
    n = R.randrange(4)
    if k == K_BYTES:
        return feature(k, [b"v" * R.randrange(5) for _ in range(n)])
    if k == K_FLOAT:
        return feature(k, [struct.pack("<f", R.random()) for _ in range(n)])
    return feature(k, [varint(R.randrange(-5, 5)) for _ in range(n)])


def _noncanon_feature(R: random.Random, f: Field, how: str) -> Tuple[bytes, str]:
    """an equivalent non-canonical Feature of a (non-FeatureList) field"""
    k, el = f.kind, f.elems
    if how == "unpacked":
        if k == K_BYTES:
            return feature(k, el), "bytes"
        mode = R.randrange(3)
        un = (lambda e: tag(1, 0) + e) if k == K_INT64 else (lambda e: tag(1, 5) + e)
        if mode == 0:
            return ld(k, b"".join(un(e) for e in el)), "unpacked"
        if mode == 1:
            return ld(k, b"".join(un(e) if i % 2 else ld(1, e) for i, e in enumerate(el))), "mixed"
        c = R.randrange(len(el) + 1)
        return ld(k, ld(1, b"".join(el[:c])) + ld(1, b"") + ld(1, b"".join(el[c:]))), "packed_segments"
    if how == "kind_twice":
        c = R.randrange(len(el) + 1)
        return ld(k, list_body(k, el[:c])) + ld(k, list_body(k, el[c:])), "kind_twice"
    if how == "oneof_decoy":
        other = R.choice([x for x in (K_BYTES, K_FLOAT, K_INT64) if x != k])
        return feature(other, elems_of(other, [1, 2] if other != K_BYTES else [b"zz"])) + feature(k, el), "oneof_decoy"
    raise ValueError(how)


def _pick(R, fs, pred=lambda f: True):
    c = [i for i, f in enumerate(fs) if pred(f)]
    return R.choice(c) if c else None


def rewrite(schema: StructType, row, record_type: int, cls: str, R: random.Random, W: int = 12,
            variant: Optional[str] = None) -> Tuple[bytes, str]:
    """-> (payload, what): a payload protobuf-java parses to the same message as `canonical(schema, row)`.  `W`: the
    parse-warp count the decoy distances are chosen for; `variant`: the key kind of class `extra` (EXTRA_KEYS), or
    "decoy_entry:<d>" for class `merge` (an earlier entry of the same key and kind, d entries in front)."""
    seq = record_type == TFR_RT_SEQUENCE_EXAMPLE
    fs = present_fields(schema, row)
    ctx_f = [f for f in fs if not f.is_flist]
    fl_f = [f for f in fs if f.is_flist]
    ctx = [entry(f.key, f.value()) for f in ctx_f]
    fls = [entry(f.key, f.value()) for f in fl_f]

    def out(c=None, l=None):
        return assemble(record_type, ctx if c is None else c, fls if l is None else l)

    if cls == "order":
        how = R.choice(["reversed", "shuffled", "rot1", "rot5", "rot7"])
        if how == "reversed":
            ctx.reverse(); fls.reverse()
        elif how == "shuffled":
            R.shuffle(ctx); R.shuffle(fls)
        else:
            k = int(how[3:])
            if ctx:
                k %= len(ctx); ctx[:] = ctx[k:] + ctx[:k]
        return out(), how
    if cls == "extra":
        variant = variant or R.choice(EXTRA_KEYS)
        key = _extra_key(R, schema, variant)
        val = _any_feature(R)
        pos = R.randrange(len(ctx) + 1)
        ctx.insert(pos, entry(key, val))
        kind = "unset" if not val else {0x0A: "bytes", 0x12: "float", 0x1A: "int64"}[val[0]]
        return out(), f"extra key {variant} ({len(key)} bytes) kind {kind} at entry {pos}"
    if cls == "null_present":
        nulls = [f for f in schema.fields if isinstance(f.dataType, NullType)]
        if not nulls:
            return out(), "no NullType field"
        f = R.choice(nulls)
        pos = R.randrange(len(ctx) + 1)
        ctx.insert(pos, entry(f.name.encode("utf-8"), _any_feature(R)))
        return out(), f"NullType {f.name} present at entry {pos}"
    if cls == "multibyte":
        key = b"mb_" + b"k" * R.choice([130, 200])
        val = feature(K_BYTES, [b"x" * R.choice([128, 300, 1000]), b"y" * 130])
        pos = R.randrange(len(ctx) + 1)
        ctx.insert(pos, entry(key, val))
        return out(), f"extra feature with multibyte lengths at entry {pos}"
    if cls == "many_entries":
        n = max(1, len(schema.fields) - len(ctx) - len(fls) + R.choice([1, 13, 40]))      # entries past the table's rows
        extra = [entry(b"x%d" % i, feature(K_INT64, [varint(i)])) for i in range(n)]
        cut = R.randrange(len(ctx) + 1)
        return out(ctx[:cut] + extra + ctx[cut:]), f"{n} extra entries at entry {cut}"
    if cls == "overlong":
        at = R.choice(["elen", "klen", "vlen", "llen", "plen", "blen", "tag"])
        i = _pick(R, ctx_f)
        if i is None:
            return out(), "no field"
        f = ctx_f[i]
        pad = R.choice([1, 2, 4])
        if at in ("plen", "blen", "llen") and not f.elems:
            at = "vlen"
        if at == "plen" and f.kind == K_BYTES:
            at = "blen"
        if at == "blen" and f.kind != K_BYTES:
            at = "plen"
        if at == "plen":
            val = ld(f.kind, ld_ov(1, b"".join(f.elems), pad))
        elif at == "blen":
            j = R.randrange(len(f.elems))
            val = ld(f.kind, b"".join(ld_ov(1, e, pad) if x == j else ld(1, e) for x, e in enumerate(f.elems)))
        elif at == "llen":
            val = ld_ov(f.kind, list_body(f.kind, f.elems), pad)
        else:
            val = f.value()
        if at == "elen":
            e = ld_ov(1, ld(1, f.key) + ld(2, val), pad)
        elif at == "klen":
            e = ld(1, ld_ov(1, f.key, pad) + ld(2, val))
        elif at == "vlen":
            e = ld(1, ld(1, f.key) + ld_ov(2, val, pad))
        elif at == "tag":
            e = ld(1, ov(0x0A, pad) + varint(len(f.key)) + f.key + ld(2, val))
        else:
            e = entry(f.key, val)
        ctx[i] = e
        return out(), f"overlong {at} (+{pad} bytes) in field {f.idx}"
    if cls == "unpacked":
        i = _pick(R, ctx_f, lambda f: f.kind != K_BYTES and len(f.elems) > 0)
        if i is None:
            return out(), "no numeric field"
        f = ctx_f[i]
        val, how = _noncanon_feature(R, f, "unpacked")
        ctx[i] = entry(f.key, val)
        return out(), f"{how} list in field {f.idx}"
    if cls == "merge":
        how = R.choice(["value_twice", "kind_twice", "oneof_decoy", "features_split", "decoy_entry"])
        if variant:
            how = variant.split(":")[0]
        if how == "features_split" or not ctx_f:
            if seq and R.random() < 0.5:
                c = R.randrange(len(fls) + 1)
                return (ld(2, b"".join(fls[:c])) + ld(1, b"".join(ctx)) + ld(2, b"".join(fls[c:]))), f"feature_lists split at {c}"
            c = R.randrange(len(ctx) + 1)
            if seq:
                return ld(1, b"".join(ctx[:c])) + ld(2, b"".join(fls)) + ld(1, b"".join(ctx[c:])), f"context split at {c}"
            return ld(1, b"".join(ctx[:c])) + ld(1, b"".join(ctx[c:])), f"features split at {c}"
        i = _pick(R, ctx_f)
        f = ctx_f[i]
        if how == "value_twice":
            c = R.randrange(len(f.elems) + 1)
            ctx[i] = ld(1, ld(1, f.key) + ld(2, feature(f.kind, f.elems[:c])) + ld(2, feature(f.kind, f.elems[c:])))
            return out(), f"value twice (split at {c}) in field {f.idx}"
        if how in ("kind_twice", "oneof_decoy"):
            val, what = _noncanon_feature(R, f, how)
            ctx[i] = entry(f.key, val)
            return out(), f"{what} in field {f.idx}"
        # an earlier entry for the same key: the later one wins.  Distance d entries before the real one: d % W == 0 puts
        # both in one parse warp, any other d in two.
        if variant:
            # same key, kind and shape (element count and string lengths), other values: only the duplicate-key check
            # tells the two entries apart
            d = int(variant.split(":")[1])
            decoy = entry(f.key, feature(f.kind, [b"d" * len(e) for e in f.elems] if f.kind == K_BYTES
                                         else elems_of(f.kind, [7] * len(f.elems))))
        else:
            d = R.choice([W, 4, 1, 5, 2 * W])
            decoy = entry(f.key, _any_feature(R, allow_unset=True))
        fill = [entry(b"fill%d" % j, feature(K_INT64, [varint(j)])) for j in range(max(0, d - 1 - i))]
        ctx[i:i] = fill
        i += len(fill)
        ctx.insert(i - (d - 1), decoy)
        return out(), f"decoy entry {d} entries before field {f.idx}{' (same kind)' if variant else ''}"
    if cls == "entry_inner":
        i = _pick(R, ctx_f)
        if i is None:
            return out(), "no field"
        f = ctx_f[i]
        if R.random() < 0.5:
            ctx[i] = ld(1, ld(2, f.value()) + ld(1, f.key))
            return out(), f"value before key in field {f.idx}"
        ctx[i] = ld(1, ld(1, b"decoy") + ld(2, f.value()) + ld(1, f.key))
        return out(), f"key twice, decoy first, in field {f.idx}"
    if cls == "unknown":
        level = R.choice(["example", "features", "entry", "feature", "list", "wrong_wiretype"])
        if level == "example":
            u = _unknowns(R)
            if seq:
                return u + ld(1, b"".join(ctx)) + _unknowns(R) + ld(2, b"".join(fls)) + _unknowns(R), "unknown fields in SequenceExample"
            return u + ld(1, b"".join(ctx)) + _unknowns(R), "unknown fields in Example"
        if level == "features":
            ctx.insert(R.randrange(len(ctx) + 1), _unknowns(R))
            return out(), "unknown fields in Features"
        i = _pick(R, ctx_f)
        if i is None:
            return out(), "no field"
        f = ctx_f[i]
        if level == "entry":
            ctx[i] = ld(1, _unknowns(R) + ld(1, f.key) + _unknowns(R) + ld(2, f.value()))
            return out(), f"unknown fields in the entry of field {f.idx}"
        if level == "feature":
            ctx[i] = entry(f.key, _unknowns(R) + f.value() + _unknowns(R))
            return out(), f"unknown fields in the Feature of field {f.idx}"
        if level == "list":
            ctx[i] = entry(f.key, ld(f.kind, _unknowns(R) + list_body(f.kind, f.elems) + _unknowns(R)))
            return out(), f"unknown fields in the list of field {f.idx}"
        # a known field number with another wire type is an unknown field
        wrong = {K_BYTES: [0, 1, 5], K_FLOAT: [0, 1, 3], K_INT64: [1, 3, 5]}[f.kind]
        u = _unknown(R, wt=R.choice(wrong), fno=1)
        ctx[i] = entry(f.key, ld(f.kind, u + list_body(f.kind, f.elems)))
        extra = tag(1, 0) + varint(7)                                       # Features.feature as a varint
        ctx.insert(R.randrange(len(ctx) + 1), extra)
        return out(), f"field 1 with a wrong wire type in Features and in the list of field {f.idx}"
    if cls == "seq":
        if not seq:
            return out(), "not a SequenceExample"
        how = R.choice(["lists_first", "omit_empty", "split_both", "flist_twice", "unknown_flist"])
        if how == "lists_first":
            return ld(2, b"".join(fls)) + ld(1, b"".join(ctx)), "feature_lists before context"
        if how == "omit_empty":
            return ((ld(1, b"".join(ctx)) if ctx else b"") + (ld(2, b"".join(fls)) if fls else b"")), "empty context / feature_lists omitted"
        if how == "split_both":
            c, d = R.randrange(len(ctx) + 1), R.randrange(len(fls) + 1)
            return (ld(1, b"".join(ctx[:c])) + ld(2, b"".join(fls[:d])) + ld(1, b"".join(ctx[c:])) + ld(2, b"".join(fls[d:]))), f"context split at {c}, feature_lists at {d}"
        i = _pick(R, fl_f)
        if i is None:
            return out(), "no FeatureList"
        f = fl_f[i]
        steps = [ld(1, feature(f.kind, s)) for s in f.steps]
        if how == "flist_twice":
            c = R.randrange(len(steps) + 1)
            fls[i] = ld(1, ld(1, f.key) + ld(2, b"".join(steps[:c])) + ld(2, b"".join(steps[c:])))
            return out(), f"FeatureList of field {f.idx} given twice (split at step {c})"
        c = R.randrange(len(steps) + 1)
        fls[i] = entry(f.key, b"".join(steps[:c]) + _unknowns(R) + b"".join(steps[c:]))
        fls.insert(R.randrange(len(fls) + 1), _unknowns(R))
        return out(), f"unknown fields in FeatureList of field {f.idx} and in FeatureLists"
    if cls == "size":
        how = R.choice(["past_64k", "big_flist", "big_cell_group"] if seq else ["past_64k", "big_cell_group"])
        if how == "past_64k":
            big = entry(b"zz_big", feature(K_BYTES, [bytes(R.randrange(256) for _ in range(64)) * 1040]))
            ctx.insert(0, big)
            return out(), "a 66 KiB feature in front of the schema's entries"
        if how == "big_flist":
            key = b"zz_flist"
            fls.insert(R.randrange(len(fls) + 1), entry(key, b"".join(ld(1, feature(K_INT64, [varint(s), varint(-s)])) for s in range(400))))
            return out(), "a 4.4 KiB FeatureList the schema does not have"
        i = _pick(R, ctx_f, lambda f: f.kind != K_BYTES and len(f.elems) > 0)
        if i is None:
            return out(), "no numeric field"
        f = ctx_f[i]
        body = b"".join(tag(1, 0 if f.kind == K_INT64 else 5) + e for e in f.elems)
        ctx[i] = ld(1, ld(1, f.key) + ld(2, ld(f.kind, ld(9, bytes(2100)) + body)))
        return out(), f"unpacked list of field {f.idx} behind 2 KiB of unknown bytes"
    raise ValueError(cls)


# --------------------------------------------------------------------------------------------
# class B: a record that fails with a known status
# --------------------------------------------------------------------------------------------
def error_record(schema: StructType, row, record_type: int, cls: str, R: random.Random, variant: Optional[str] = None):
    """-> (payload, code, field, what) or None when the schema cannot express this error.  The rest of the record is
    valid, so the first error in schema order is the constructed one.  `variant`: the MAL_SHAPES name of class
    `malformed`; "feature" (a 2-D field fed from a Feature) or "flist" (a scalar fed from a FeatureList) of class
    `bad_nesting`."""
    seq = record_type == TFR_RT_SEQUENCE_EXAMPLE
    fs = present_fields(schema, row)
    ctx_f = [f for f in fs if not f.is_flist]
    fl_f = [f for f in fs if f.is_flist]
    ctx = [entry(f.key, f.value()) for f in ctx_f]
    fls = [entry(f.key, f.value()) for f in fl_f]
    out = lambda: assemble(record_type, ctx, fls)
    if cls in ("kind_mismatch", "kind_not_set"):
        i = _pick(R, ctx_f)
        if i is None:
            return None
        f = ctx_f[i]
        if cls == "kind_not_set":
            ctx[i] = entry(f.key, b"")
        else:
            other = R.choice([x for x in (K_BYTES, K_FLOAT, K_INT64) if x != f.kind])
            ctx[i] = entry(f.key, feature(other, elems_of(other, [3] if other != K_BYTES else [b"q"]) * R.randrange(2)))
        return out(), A.TFR_E_KIND_MISMATCH, f.idx, f"{cls} in field {f.idx}"
    if cls == "empty_scalar":
        i = _pick(R, ctx_f, lambda f: not isinstance(schema.fields[f.idx].dataType, ArrayType))
        if i is None:
            return None
        f = ctx_f[i]
        ctx[i] = entry(f.key, feature(f.kind, []))
        return out(), A.TFR_E_EMPTY_SCALAR, f.idx, f"empty list for scalar field {f.idx}"
    if cls == "null_in_nonnull":
        i = _pick(R, ctx_f, lambda f: not schema.fields[f.idx].nullable)
        if i is None:
            return None
        f = ctx_f.pop(i)
        ctx.pop(i)
        return out(), A.TFR_E_NULL_IN_NONNULL, f.idx, f"non-nullable field {f.idx} missing"
    if cls == "bad_nesting":
        if not seq:
            two_d = [i for i, f in enumerate(schema.fields)
                     if isinstance(f.dataType, ArrayType) and isinstance(f.dataType.elementType, ArrayType)]
            if not two_d or variant == "flist":
                return None
            i = R.choice(two_d)                            # an Example can only give a 2-D field a Feature
            ctx.insert(R.randrange(len(ctx) + 1), entry(schema.fields[i].name.encode("utf-8"), feature(K_INT64, [varint(5)])))
            return out(), A.TFR_E_BAD_NESTING, i, f"2-D field {i} from a Feature"
        if fl_f and (variant == "feature" or (variant is None and R.random() < 0.5)):     # a 2-D field fed from a Feature
            i = R.randrange(len(fl_f))
            f = fl_f[i]
            fls.pop(i)
            ctx.insert(R.randrange(len(ctx) + 1), entry(f.key, feature(f.kind, f.steps[0] if f.steps else [])))
            return out(), A.TFR_E_BAD_NESTING, f.idx, f"2-D field {f.idx} from a Feature"
        i = _pick(R, ctx_f, lambda f: not isinstance(schema.fields[f.idx].dataType, ArrayType))
        if i is None:
            return None
        f = ctx_f[i]                                       # a scalar fed from a FeatureList
        ctx.pop(i)
        fls.insert(R.randrange(len(fls) + 1), entry(f.key, ld(1, f.value())))
        return out(), A.TFR_E_BAD_NESTING, f.idx, f"scalar field {f.idx} from a FeatureList"
    if cls == "malformed":
        name = variant or R.choice(sorted(MAL_SHAPES))
        return out() + MAL_SHAPES[name], A.TFR_E_MALFORMED_PROTO, -1, name
    if cls in ("groups_24", "groups_25"):
        d = int(cls[-2:])
        # protobuf-java skips both (its limit is 100 nested messages); the GPU parsers match groups with a 24-deep stack
        # and report deeper nesting as malformed (the documented deviation, DESIGN §2): the code here is Java's
        g = b"".join(tag(5 + k, 3) for k in range(d)) + tag(99, 0) + varint(1) + b"".join(tag(5 + k, 4) for k in reversed(range(d)))
        return g + out(), 0, -1, f"unknown group nested {d} deep"
    raise ValueError(cls)


def two_errors_in_one_record(schema: StructType, row, record_type: int, R: random.Random):
    """two fields fail; the later one in schema order comes first on the wire.  -> (payload, code, field, what) of the
    error the reference reports (the first in schema order) or None"""
    fs = present_fields(schema, row)
    ctx_f = [f for f in fs if not f.is_flist]
    if len(ctx_f) < 2:
        return None
    i, j = sorted(R.sample(range(len(ctx_f)), 2))
    fi, fj = ctx_f[i], ctx_f[j]
    bad = lambda f: entry(f.key, feature(K_BYTES if f.kind != K_BYTES else K_INT64, []))
    ents = [entry(f.key, f.value()) for f in ctx_f]
    ents[i], ents[j] = bad(fj), bad(fi)                   # wire order: field j's bad entry, then field i's
    fls = [entry(f.key, f.value()) for f in fs if f.is_flist]
    return assemble(record_type, ents, fls), A.TFR_E_KIND_MISMATCH, fi.idx, f"kind mismatch in fields {fi.idx} and {fj.idx}"


# --------------------------------------------------------------------------------------------
# class C: byte-wise damage (the CRC is recomputed)
# --------------------------------------------------------------------------------------------
def mutate(payload: bytes, R: random.Random) -> Tuple[bytes, str]:
    b = bytearray(payload)
    how = R.choice(["flip", "insert", "delete", "overwrite"]) if b else "insert"
    pos = R.randrange(len(b) + (1 if how == "insert" else 0))
    if how == "flip":
        b[pos] ^= 1 << R.randrange(8)
    elif how == "insert":
        b[pos:pos] = bytes(R.randrange(256) for _ in range(R.randrange(1, 4)))
    elif how == "delete":
        del b[pos:pos + R.randrange(1, 4)]
    else:
        n = R.randrange(1, 5)
        b[pos:pos + n] = bytes(R.randrange(256) for _ in range(len(b[pos:pos + n])))
    return bytes(b), f"{how} at byte {pos}"


# --------------------------------------------------------------------------------------------
# known deviations of upb from protobuf-java (for the differential checks against upb)
# --------------------------------------------------------------------------------------------
def _read_varint(b, p):
    v, s = 0, 0
    while True:
        if p >= len(b) or s > 63:
            raise ValueError
        c = b[p]; p += 1
        v |= (c & 0x7F) << s; s += 7
        if c < 0x80:
            return v, p


def _fields(b):
    """(field number, wire type, payload) of a message's fields; raises ValueError when they do not parse"""
    p, out = 0, []
    while p < len(b):
        t, p = _read_varint(b, p)
        fno, wt = t >> 3, t & 7
        if wt == 2:
            n, p = _read_varint(b, p)
            if p + n > len(b):
                raise ValueError
            out.append((fno, wt, b[p:p + n])); p += n
        elif wt == 0:
            _, p = _read_varint(b, p); out.append((fno, wt, None))
        elif wt in (1, 5):
            p += 8 if wt == 1 else 4
            if p > len(b):
                raise ValueError
            out.append((fno, wt, None))
        else:
            out.append((fno, wt, None))
            return out                                     # groups: not followed here
    return out


def _long_tag(b: bytes, depth: int = 0) -> bool:
    """a field tag of more than five varint bytes in `b` or in any length-delimited field that parses as a message"""
    p = 0
    try:
        while p < len(b):
            q = p
            t, p = _read_varint(b, p)
            if p - q > 5:
                return True
            wt = t & 7
            if wt == 2:
                n, p = _read_varint(b, p)
                if depth < 8 and _long_tag(b[p:p + n], depth + 1):
                    return True
                p += n
            elif wt == 0:
                _, p = _read_varint(b, p)
            elif wt in (1, 5):
                p += 8 if wt == 1 else 4
    except ValueError:
        pass
    return False


def upb_deviation(payload: bytes, record_type: int) -> Optional[str]:
    """the known reason why upb may disagree with protobuf-java on this payload, or None:
      * upb keeps a map entry that carries an unknown field as an unknown field of the map (its key and value are then
        never looked at), protobuf-java skips the unknown field and puts the entry;
      * upb rejects a field tag longer than five varint bytes, protobuf-java's readTag keeps its low 32 bits."""
    if _long_tag(payload):
        return "tag longer than five bytes"
    try:
        top = _fields(payload)
    except ValueError:
        return None
    maps = []
    for fno, wt, body in top:
        if wt != 2:
            continue
        if fno == 1 or (record_type == TFR_RT_SEQUENCE_EXAMPLE and fno == 2):
            maps.append(body)
    for m in maps:
        try:
            ents = _fields(m)
        except ValueError:
            continue
        for fno, wt, body in ents:
            if fno != 1 or wt != 2:
                continue
            try:
                inner = _fields(body)
            except ValueError:
                return "map entry that does not parse"
            if any(not (f in (1, 2) and w == 2) for f, w, _ in inner):
                return "unknown field inside a map entry"
    return None
