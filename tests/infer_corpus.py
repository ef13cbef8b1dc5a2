"""Seeded corpora for schema inference (tfr_infer_*, DESIGN §9).  TEST INFRASTRUCTURE ONLY.

Records are built directly on the wire, with no schema, so that a map can hold what no writer produces: a key twice
with the error in the overwritten entry, the surviving one or both; an entry without a key or with unknown fields;
`features` / `context` / `feature_lists` split over several top-level fields, `context` after `feature_lists`; two
errors in one record, in either map and either order.  Inference (M/TensorFlowInferSchema.scala) takes each map in its
order (the position of each key's first occurrence, Map.put keeps it), context before feature_lists, and stops at the
first error; a malformed record fails in parseFrom before inference sees a value.

Names: empty, 1 and 300 bytes, multibyte UTF-8, shared prefixes, and COLL_A / COLL_B, two different 16-byte names with
the same 64-bit FNV-1a hash (the hash the GPU table is keyed by).

`batch(seed, rt, n)` returns one Batch: the payloads, the framed bytes (a data CRC flipped or the final frame truncated
in some batches) and a note of what was put where, for failure messages.  `payload_table()` holds the hand-written
regressions whose verdicts are pinned on the CPU."""
from __future__ import annotations

import random
import struct
from typing import List, Optional

from oracle import pyref
from oracle.pyref import ld, map_entry, tag, varint
from spark_tfrecord_b200 import _cabi as A

COLL_A, COLL_B = b"7394ab0f5939e582", b"76ebcdcca5eca4fb"


def fnv1a64(b: bytes) -> int:
    h = 1469598103934665603
    for c in b:
        h = ((h ^ c) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


assert COLL_A != COLL_B and fnv1a64(COLL_A) == fnv1a64(COLL_B) == 0x72FF70D38778656F

FIXED_NAMES = [b"", b"x", b"n" * 300, "ключ".encode(), "キー😀".encode(), "é".encode(), "中文字段名".encode(),
               b"pre", b"pre_", b"pre_a", b"pre_ab", COLL_A, COLL_B]


# --------------------------------------------------------------------------------------------
# values
# --------------------------------------------------------------------------------------------
def i64(*v) -> bytes:
    return ld(3, ld(1, b"".join(varint(x) for x in v)))


def f32(*v) -> bytes:
    return ld(2, ld(1, b"".join(struct.pack("<f", x) for x in v)))


def byt(*v) -> bytes:
    return ld(1, b"".join(ld(1, x) for x in v))


def fl(*steps) -> bytes:
    """a FeatureList of these steps (each a Feature; b"" is a step whose kind is not set)"""
    return b"".join(ld(1, s) for s in steps)


UNSET = b""                      # a Feature whose kind is not set


def feature(R: random.Random, n: Optional[int] = None, kind: Optional[str] = None) -> bytes:
    """a Feature of a set kind with a list of 0, 1 or several values, in one of several wire forms"""
    kind = kind or R.choice("ifb")
    n = R.choice([0, 1, 1, 2, 5]) if n is None else n
    if kind == "i":
        vals = [R.choice([0, 1, -1, 300, 2**63 - 1]) for _ in range(n)]
        if n == 0 and R.random() < 0.5:
            return ld(3, b"")                                      # an Int64List with no field at all
        if R.random() < 0.3:
            return ld(3, b"".join(tag(1, 0) + varint(v) for v in vals))      # unpacked
        return i64(*vals)
    if kind == "f":
        vals = [R.choice([0.0, 1.5, -2.0]) for _ in range(n)]
        if n == 0 and R.random() < 0.5:
            return ld(2, b"")
        return f32(*vals)
    vals = [R.choice([b"", b"s", "é".encode(), b"z" * 40]) for _ in range(n)]
    return byt(*vals)


EMPTY_STEPS = [b"steps_empty_a", b"steps_empty_b"]     # the only names of FeatureLists whose steps are all empty


def empty_steps(R: random.Random) -> bytes:
    """a FeatureList of 1-3 empty steps: ArrayType(ArrayType(null)), code 10, which merges with nothing but null"""
    return fl(*(feature(R, 0) for _ in range(R.randrange(1, 4))))


def flist(R: random.Random) -> bytes:
    """a valid FeatureList: 1-4 steps of one kind or of mixed kinds, lists of 0, 1 or several values"""
    steps = R.randrange(1, 5)
    kinds = R.choice(["same", "mixed"])
    k = R.choice("ifb")
    full = R.randrange(steps)                                      # one step holds a value: not all empty
    return fl(*(feature(R, R.choice([1, 3]) if s == full else None, k if kinds == "same" else None) for s in range(steps)))


# --------------------------------------------------------------------------------------------
# map entries
# --------------------------------------------------------------------------------------------
def unknown(R: random.Random) -> bytes:
    """an unknown field (field numbers 3..9 are unknown in every message here)"""
    f = R.randrange(3, 10)
    w = R.choice([0, 1, 2, 5, 3])
    if w == 0:
        return tag(f, 0) + varint(R.choice([0, 300, 2**64 - 1]))
    if w == 1:
        return tag(f, 1) + bytes(8)
    if w == 2:
        return ld(f, b"u" * R.choice([0, 3, 130]))
    if w == 5:
        return tag(f, 5) + bytes(4)
    return tag(f, 3) + tag(f + 1, 0) + varint(1) + tag(f, 4)      # a group with one field


def entry(R: random.Random, key: bytes, value: bytes, style: str = "plain") -> bytes:
    if style == "nokey":
        return ld(1, ld(2, value))                                 # the key is ""
    if style == "value_first":
        return ld(1, ld(2, value) + ld(1, key))
    if style == "unknown":
        return ld(1, unknown(R) + ld(1, key) + ld(2, value) + unknown(R))
    if style == "key_twice":
        return ld(1, ld(1, b"decoy") + ld(2, value) + ld(1, key))
    return map_entry(key, value)


class Ent:
    __slots__ = ("key", "value", "style", "note")

    def __init__(self, key, value, style="plain", note=""):
        self.key, self.value, self.style, self.note = key, value, style, note


def _bad_value(R: random.Random, is_flist: bool, kind: str) -> bytes:
    if kind == "kind_not_set":
        return fl(*([feature(R)] * R.randrange(2) + [UNSET])) if is_flist else UNSET
    assert kind == "empty_flist" and is_flist
    return b""


MALFORMED = {      # bytes that make the map (or top level) they sit in fail to parse
    "trunc_len": bytes([0x0A, 0x05, 0x01]),                        # an entry whose length runs past its map
    "bad_group": tag(5, 3) + tag(6, 0) + varint(1),                # a group that never ends
    "bad_end_group": tag(5, 3) + tag(6, 4),                        # a group closed by another field number
}
VALUE_ERRORS = ["kind_not_set", "empty_flist"]
ERRORS = VALUE_ERRORS + list(MALFORMED)
PLACES = ["overwritten", "surviving", "both", "alone"]


# upb keeps a map entry that carries an unknown field as an unknown field of the map and never looks at its key or
# value; protobuf-java skips the unknown field and puts the entry
UPB_DEVIATES = "an entry with unknown fields"


class Rec:
    """one record under construction: its maps as entry lists, then the wire form"""

    def __init__(self, R: random.Random, rt: int, names: List[bytes]):
        self.R, self.rt, self.names = R, rt, names
        self.maps = [[], []]                                       # context/features, feature_lists
        self.trailer = [b"", b""]                                  # raw bytes at the end of a map body
        self.top_trailer = b""
        self.notes = []

    def fill(self, n_ctx: int, n_fl: int):
        R = self.R
        for m, n in ((0, n_ctx), (1, n_fl if self.rt == 1 else 0)):
            for _ in range(n):
                key = R.choice(self.names)
                val = flist(R) if m else feature(R)
                if m and R.random() < 0.1:
                    key, val = R.choice(EMPTY_STEPS), empty_steps(R)
                style = R.choices(["plain", "nokey", "value_first", "unknown", "key_twice"], [20, 1, 1, 1, 1])[0]
                if style == "nokey" and key in EMPTY_STEPS:
                    style = "plain"
                self.maps[m].append(Ent(key if style != "nokey" else b"", val, style))
        return self

    def duplicate(self, m: int, dist: int):
        """the key of one entry again, `dist` entries later (filled up with fresh keys); the later one wins"""
        R, ents = self.R, self.maps[m]
        if not ents:
            return
        i = R.randrange(len(ents))
        while len(ents) < i + dist + 1:
            ents.append(Ent(R.choice(self.names) + b"_f%d" % len(ents), flist(R) if m else feature(R)))
        j = i + dist + 1
        val = (empty_steps(R) if ents[i].key in EMPTY_STEPS else flist(R)) if m else feature(R)
        ents.insert(j, Ent(ents[i].key, val, "plain", f"dup of entry {i}"))
        self.notes.append(f"map {m}: key {ents[i].key[:20]!r} again at distance {dist}")

    def error(self, m: int, kind: str, place: str = "alone"):
        R, ents = self.R, self.maps[m]
        if kind in MALFORMED:
            where = R.choice(["map", "top", "value"]) if ents else R.choice(["map", "top"])
            if where == "map":
                self.trailer[m] += MALFORMED[kind]
            elif where == "top":
                self.top_trailer += MALFORMED[kind]
            else:
                e = R.choice(ents)
                e.value = e.value + (MALFORMED[kind] if not m else ld(1, MALFORMED[kind]))
            self.notes.append(f"{kind} in {where} of map {m}")
            return
        if kind == "empty_flist" and m == 0:
            kind = "kind_not_set"
        key = R.choice(self.names) + b"_e%d" % R.randrange(1000)
        good = lambda: flist(R) if m else feature(R)
        bad = lambda: _bad_value(R, m == 1, kind)
        pos = R.randrange(len(ents) + 1)
        d = R.choice([0, 1, 31, 32, 33, 70])
        if place == "alone":
            seq = [Ent(key, bad())]
        elif place == "overwritten":
            seq = [Ent(key, bad())] + [Ent(key + b"_g%d" % k, good()) for k in range(d)] + [Ent(key, good())]
        elif place == "surviving":
            seq = [Ent(key, good())] + [Ent(key + b"_g%d" % k, good()) for k in range(d)] + [Ent(key, bad())]
        else:
            seq = [Ent(key, bad())] + [Ent(key + b"_g%d" % k, good()) for k in range(d)] + [Ent(key, bad())]
        ents[pos:pos] = seq
        self.notes.append(f"{kind} {place} (distance {d}) at entry {pos} of map {m}")

    def payload(self) -> bytes:
        R = self.R
        if any(e.style == "unknown" for m in self.maps for e in m):
            self.notes.append(UPB_DEVIATES)
        bodies = []
        for m in (0, 1):
            if m == 1 and self.rt != 1:
                break
            parts = [entry(R, e.key, e.value, e.style) for e in self.maps[m]]
            if parts and R.random() < 0.1:
                parts.insert(R.randrange(len(parts) + 1), tag(2, 0) + varint(7))     # an unknown field in the map
            # a repeated top-level field merges: the map split over 1-3 fields
            cuts = sorted(R.sample(range(len(parts) + 1), min(len(parts) + 1, R.choice([1, 1, 1, 2, 3]) - 1)))
            segs, prev = [], 0
            for c in cuts + [len(parts)]:
                segs.append(b"".join(parts[prev:c]))
                prev = c
            segs[-1] += self.trailer[m]
            bodies.append([ld(m + 1, s) for s in segs if s or R.random() < 0.5 or s is segs[-1]])
        if self.rt == 1 and R.random() < 0.3:
            bodies.reverse()                                       # context after feature_lists
        fields = [f for b in bodies for f in b]
        if len(bodies) == 2 and R.random() < 0.2:
            R.shuffle(fields)                                      # interleaved
        if R.random() < 0.1:
            fields.insert(R.randrange(len(fields) + 1), unknown(R))
        return b"".join(fields) + self.top_trailer


# --------------------------------------------------------------------------------------------
# batches
# --------------------------------------------------------------------------------------------
class Batch:
    def __init__(self, rt, payloads, notes, crc_row=None, truncated=False):
        self.rt, self.payloads, self.notes = rt, payloads, notes
        self.crc_row, self.truncated = crc_row, truncated
        frames = [pyref.frame_fast(p) for p in payloads]
        if crc_row is not None:
            f = bytearray(frames[crc_row])
            f[-1 - (crc_row % 4)] ^= 0x10                          # the stored data CRC no longer matches
            frames[crc_row] = bytes(f)
        self.frame_ends = []
        pos = 0
        for f in frames:
            pos += len(f)
            self.frame_ends.append(pos)
        data = b"".join(frames)
        if truncated:
            last = len(frames[-1])
            data = data[:len(data) - last + _kept_bytes(len(payloads), last)]
            self.frame_ends.pop()
        self.data = data

    def describe(self) -> str:
        s = [f"rt {self.rt}, {len(self.payloads)} records"]
        if self.crc_row is not None:
            s.append(f"data CRC flipped in record {self.crc_row}")
        if self.truncated:
            s.append("final frame truncated")
        s += [f"record {r}: {n}" for r, n in self.notes]
        return "; ".join(s)


def _kept_bytes(seed: int, frame_len: int) -> int:
    """bytes of the final frame that are kept: past its 12-byte header, short of its end"""
    return 12 + seed % (frame_len - 12)


def names_pool(R: random.Random, k: int) -> List[bytes]:
    out = list(FIXED_NAMES)
    while len(out) < k:
        out.append(R.choice([b"f", b"feat_", "名".encode(), b"pre_a"]) + str(len(out)).encode())
    return out


MODES = ["clean", "clean", "one", "two_in_record", "two_records", "crc", "truncated", "conflict"]


def record(R: random.Random, rt: int, names: List[bytes], errors=()) -> (bytes, str):
    wide = R.random() < 0.08
    n_ctx = R.randrange(40, 110) if wide else R.randrange(0, 8)
    n_fl = R.randrange(40, 110) if wide and R.random() < 0.5 else R.randrange(0, 6)
    r = Rec(R, rt, names).fill(n_ctx, n_fl)
    if R.random() < 0.3:
        r.duplicate(R.randrange(2 if rt == 1 else 1), R.choice([0, 31, 32, 33, 70]))
    for kind, m, place in errors:
        r.error(m, kind, place)
    return r.payload(), "; ".join(r.notes)


def _rand_error(R, rt):
    kind = R.choices(ERRORS, [3, 2, 1, 1, 1])[0]
    m = R.randrange(2) if rt == 1 else 0
    if kind == "empty_flist" and m == 0:
        kind = "kind_not_set"
    return kind, m, R.choice(PLACES)


def batch(seed: int, rt: int, n: int, mode: Optional[str] = None) -> Batch:
    """`n` records of record type `rt`; `mode` (default: drawn from MODES by the seed) says where errors go"""
    R = random.Random(f"infer/{seed}/{rt}/{n}")
    mode = mode or MODES[seed % len(MODES)]
    names = names_pool(R, R.choice([20, 60, 400]))
    errs = {}
    if mode == "one":
        errs[R.randrange(n)] = [_rand_error(R, rt)]
    elif mode == "two_in_record":
        errs[R.randrange(n)] = [_rand_error(R, rt), _rand_error(R, rt)]
    elif mode == "two_records":
        for r in R.sample(range(n), min(2, n)):
            errs[r] = [_rand_error(R, rt)]
    payloads, notes = [], []
    for row in range(n):
        p, note = record(R, rt, names, errs.get(row, ()))
        payloads.append(p)
        if note:
            notes.append((row, note))
    if mode == "conflict" and rt == 1 and n >= 2:
        # a name of all-empty steps in one record is a FeatureList of Longs in another: UNSUPPORTED_TYPE once they merge
        r1, r2 = R.sample(range(n), 2)
        key = R.choice(EMPTY_STEPS)
        payloads[r1] = ld(2, map_entry(key, empty_steps(R)))
        payloads[r2] = ld(1, map_entry(b"c", i64(2))) + ld(2, map_entry(key, fl(i64(1), feature(R, 0))))
        notes += [(r1, f"{key!r}: all steps empty"), (r2, f"{key!r}: steps of Longs")]
    crc_row = R.randrange(n) if mode == "crc" else None
    return Batch(rt, payloads, notes, crc_row, mode == "truncated" and n > 0)


def payload_table():
    """the hand-written regressions: (name, payload, record type, the oracle's status, its names -> codes)"""
    a, b, c, e = b"a", b"b", b"c", b"e"
    return [
        ("error_in_overwritten_entry", ld(1, map_entry(a, UNSET) + map_entry(a, i64(1))), 0, 0, {a: 1}),
        ("malformed_after_value_error", ld(1, map_entry(a, UNSET) + map_entry(b, i64(1))) + b"\x0a\x05\x01", 0,
         A.TFR_E_MALFORMED_PROTO, None),
        ("empty_flist_overwritten", ld(2, map_entry(e, b"") + map_entry(e, fl(i64(1)))), 1, 0, {e: 7}),
        ("first_error_in_map_order", ld(2, map_entry(a, fl(UNSET)) + map_entry(b, b"")), 1, A.TFR_E_KIND_MISMATCH, None),
        ("malformed_feature_lists_after_context_error", ld(1, map_entry(c, UNSET)) + ld(2, b"\x0a\x03\x0a\x09\x00"), 1,
         A.TFR_E_MALFORMED_PROTO, None),
        ("equal_hash_names", ld(1, map_entry(COLL_A, i64(1)) + map_entry(COLL_B, ld(1, ld(1, b"s")))), 0, 0,
         {COLL_A: 1, COLL_B: 3}),
    ]
