"""Non-canonical, CRC-valid wire forms through every decode path, one mutated record per batch, against the oracle.

The tile kernel (tile.cuh) takes only the writer's canonical shape and flags everything else, which sends the WHOLE batch
to the general kernels (decode.cuh).  A record it rejects correctly would hide a wrong acceptance of another record of
the same batch, so every batch here holds exactly one rewritten record among the writer's canonical ones, at row 0, 31,
32 (the tile boundary), a middle row or the last row.  The rewrites are tests/wire_rewrite.py's classes:
  A  equivalent rewrites: the rows must be the source rows.  Every class twice at random, and on every schema every
     extra-key kind and an earlier entry of the same key AND kind at a distance of 4, 12 (same parse warp for the
     4 + 1 and the 12 + 3 kernels: the per-warp `seen` bits), 1 and 5 (two warps: the shared `sseen` merge);
  B  errors with a valid CRC: kind mismatch, kind not set, .head of an empty list, a missing non-nullable field, bad
     nesting (both ways), EVERY malformed shape of wire_rewrite.MAL_SHAPES, unknown groups nested 24 and 25 deep, two
     errors in a batch / in a record;
  C  byte-wise damage with the CRC recomputed (differential only).
Each mutated batch goes through
  1. `Decoder.decode` of a fresh decoder (its first batch: the synchronising decode, count mode);
  2. `Decoder.submit` of a decoder in its steady state (see MODES);
  3. a decoder created with TFR_DISABLE_FAST=1 (the general kernels only);
  4. `Infer.update`, against `oracle.infer`.
Every decode must equal the oracle's decode of the same bytes in error code, row and field, rows, consumed bytes and every
column.  Canonical rewrites (CANONICAL_CLASSES: entry order, extra features, a present NullType field, multibyte
lengths, more entries than the entry table has rows) must stay on the fast path: a regression there is a silent
performance cliff on files written by TensorFlow (C++ protobuf writes map entries in hash order).  A record larger than
every slot learned so far is redone once (then the same bytes must stay on the fast path).  After every mutated batch a
clean batch must be decoded in the configuration's steady state again.

MODES, the steady state each configuration is asserted to be in (`Decoder.stats()` around every clean and canonical
batch):
  pipelined  speculative submit, one more `speculative_submits` (plus one per rerun in the transcoding instantiation),
             nothing redone, nothing on the general path.  All Example schemas of <= 128 fields without a 2-D column:
             uniform (all lists of one length), one-pass ragged, and -- w12_small_ragged_utf8, whose ragged string column
             carries malformed UTF-8 -- the transcoding instantiation (`transcode_reruns` >= 1 is asserted); and the
             SequenceExample schemas seq12_uniform and seq5_ragged (<= 4 variable-width columns, FeatureLists of numbers).
  sync       the synchronising decode through the tile kernel, never speculative: seq13_big_ragged, seq40_ragged and
             seq65_ragged.  Their FeatureList columns hold strings or come with more than 4 variable-width columns,
             which the pipelined SequenceExample kernel does not keep per-step counts for (api_decode.inc: learn_shapes).
  general    every batch on the general path: schemas of more than 128 fields (w129, w300) and an Example schema with an
             array<array<>> column (w12_ex_2d), which the tile kernel does not take (api_decode.inc: the fast path's
             eligibility).
Two size limits put records on the general path whatever their shape, asserted as such:
  * a payload over 64 KiB (class `size`, "a 66 KiB feature"): the synchronising decode sizes a tile as 32 slots of the
    largest record, which no shared memory holds; the pipelined tile, sized from the previous batch, overflows and the
    batch is redone through the synchronising decode.  The tile kernel's 16-bit entry table limit (entries past 64 KiB)
    is therefore out of reach of any batch that gets to the tile kernel;
  * the same 32-slot sizing of the synchronising decode caps a record at about 6 KB on a 128-field schema (the schema's
    constants and entry table share the 227 KB): class `many_entries` keeps to 1, 13 or 40 entries past the table so
    that its records stay under it.
The one documented deviation (DESIGN §2): unknown groups nested deeper than 24 are malformed on the GPU, while
protobuf-java skips them.
Reference semantics: M/TFRecordDeserializer.scala:21-61,68-143, M/TensorFlowInferSchema.scala."""
import os
import random

import numpy as np
import pytest

import wire_rewrite as W
from oracle import pyref
from util import assert_columns_equal, slice_columns
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


# (name, width, record type, make_schema options, steady-state mode)
# Small records (tens of bytes) make the tile kernel take its 4 + 1 warp geometry, ~2 KiB records the 12 + 3 one.
CONFIGS = [
    ("w1_small", 1, 0, dict(uniform=True), "pipelined"),
    ("w12_small_uniform", 12, 0, dict(uniform=True), "pipelined"),
    ("w12_small_ragged", 12, 0, dict(), "pipelined"),
    ("w12_small_ragged_utf8", 12, 0, dict(bad_utf8=True), "pipelined"),
    ("w13_big_uniform", 13, 0, dict(big=True, uniform=True), "pipelined"),
    ("w13_big_ragged", 13, 0, dict(big=True), "pipelined"),
    ("w63_ragged", 63, 0, dict(), "pipelined"),
    ("w64_uniform", 64, 0, dict(uniform=True), "pipelined"),
    ("w65_ragged", 65, 0, dict(), "pipelined"),
    ("w127_uniform", 127, 0, dict(uniform=True), "pipelined"),
    ("w128_ragged", 128, 0, dict(big=True), "pipelined"),
    ("w129_ragged", 129, 0, dict(), "general"),
    ("w300_uniform", 300, 0, dict(uniform=True), "general"),
    ("w12_ex_2d", 12, 0, dict(with_2d=True), "general"),
    ("seq12_uniform", 12, 1, dict(uniform=True), "pipelined"),
    ("seq5_ragged", 5, 1, dict(flist_numeric=True), "pipelined"),
    ("seq13_big_ragged", 13, 1, dict(big=True), "sync"),
    ("seq40_ragged", 40, 1, dict(), "sync"),
    ("seq65_ragged", 65, 1, dict(), "sync"),
]
DECOY_DISTANCES = [4, 12, 1, 5]


def in_mode(mode, s0, s1, bad_utf8=False):
    """the batch between the stats s0 and s1 was decoded the way `mode` says (see the module docstring)"""
    d = {k: s1[k] - s0[k] for k in s0}
    if mode == "general":
        return d["general_path_batches"] == 1
    if d["speculative_redone"] or d["general_path_batches"]:
        return False
    if mode == "sync":
        return d["speculative_submits"] == 0 and d["batches"] == 1
    return d["speculative_submits"] == 1 + d["transcode_reruns"]


class Want:
    def __init__(self, info, columns):
        self.info, self.columns = info, columns


def _hex(p: bytes) -> str:
    h = p.hex()
    return h if len(h) <= 4096 else h[:4096] + f"... ({len(p)} bytes)"


class Harness:
    def __init__(self, native, oracle, cfg):
        self.native, self.oracle = native, oracle
        self.name, self.width, self.rt, opts, self.mode = cfg
        self.bad_utf8 = bad_utf8 = opts.get("bad_utf8", False)
        self.seed = sum(map(ord, self.name))
        self.sch, gen = W.make_schema(self.seed, self.width, self.rt, **opts)
        r = np.random.default_rng(self.seed + 1)
        rows = [gen(r) for _ in range(64)]
        mean = np.mean([len(W.canonical(self.sch, row, self.rt)) for row in rows])
        self.n = max(96, int(24576 / (mean + 16)) + 1)      # (a batch of 64 records or fewer teaches the decoder no sizes)
        rows += [gen(r) for _ in range(self.n - 64)]
        self.rows = rows
        self.framed = [pyref.frame_fast(W.canonical(self.sch, row, self.rt)) for row in rows]
        self.clean = np.frombuffer(b"".join(self.framed), np.uint8)
        self.want_clean = oracle.decode(self.clean, self.sch, self.rt)
        assert self.want_clean.info["error_code"] == 0 and self.want_clean.n_rows == self.n, self.want_clean.info
        if not bad_utf8:
            assert_columns_equal(self.want_clean.columns, W.source_columns(self.sch, rows, self.rt), self.sch.names,
                                 f"{self.name}: oracle vs source")
        self.dec = native.Decoder(self.sch, self.rt)
        os.environ["TFR_DISABLE_FAST"] = "1"
        try:
            self.gen_dec = native.Decoder(self.sch, self.rt)
        finally:
            del os.environ["TFR_DISABLE_FAST"]
        # the shapes are learned from a batch without malformed UTF-8 (a batch with it goes to the general path, which
        # learns nothing); the pipelined batches then run the transcoding instantiation of the tile kernel
        learn = [tuple([("ok" if isinstance(x, bytes) else x) for x in v] if bad_utf8 and j == 2 and v is not None else v
                       for j, v in enumerate(row)) for row in rows]
        learn = np.frombuffer(W.frame(W.canonical(self.sch, row, self.rt) for row in learn), np.uint8)
        b, _ = self.dec.decode(learn)
        self.check(b, self.oracle.decode(learn, self.sch, self.rt), "learning batch"); b.release()
        self.clean_submit("steady state", True)

    def close(self):
        self.dec.close()
        self.gen_dec.close()

    def check(self, b, want, what):
        info = b.info
        for k in ("error_code", "error_row", "error_field", "n_rows", "consumed_bytes"):
            assert info[k] == want.info[k], f"{what}: {k} {info[k]} != {want.info[k]} (got {info}, want {want.info})"
        assert_columns_equal(b.to_host(), want.columns, self.sch.names, what)

    def clean_submit(self, what, assert_steady):
        s0 = self.dec.stats()
        b = self.dec.submit(self.clean)
        self.check(b, self.want_clean, f"{self.name}: clean batch after {what}"); b.release()
        s1 = self.dec.stats()
        if assert_steady:
            assert in_mode(self.mode, s0, s1), f"{self.name}: clean batch after {what} not decoded {self.mode}: {s0} -> {s1}"

    def run(self, cls, payload, row, what, code=None, field=None, more=()):
        """one batch: the canonical records with `payload` at `row` (and the (row, payload) pairs of `more`)"""
        fr = list(self.framed)
        fr[row] = pyref.frame_fast(payload)
        for r2, p2 in more:
            fr[r2] = pyref.frame_fast(p2)
        data = np.frombuffer(b"".join(fr), np.uint8)
        tag = f"[{self.name} seed {self.seed} width {self.width} rt {self.rt}] class {cls} ({what}) at row {row}"
        msg = f"{tag}; payload {_hex(payload)}"
        want = self.oracle.decode(data, self.sch, self.rt)
        if cls in W.A_CLASSES:
            assert want.info["error_code"] == 0, (msg, want.info)
            assert_columns_equal(want.columns, self.want_clean.columns, self.sch.names, f"oracle, {msg}")
        elif code is not None:
            if code:
                assert (want.info["error_code"], want.info["error_row"], want.info["error_field"]) == (code, row, field), (msg, want.info)
            else:
                assert want.info["error_code"] == 0, (msg, want.info)
        infer_rc = None
        if cls == "groups_25":
            # the documented deviation: a 25-deep group stack is malformed on the GPU, the rows before it stand
            info = dict(want.info, error_code=A.TFR_E_MALFORMED_PROTO, error_row=row, error_field=-1, n_rows=row)
            info["consumed_bytes"] = sum(len(f) for f in fr[:row])
            want = Want(info, slice_columns(want.columns, 0, row))
            # inference stops at the first failing record: an earlier one's status, or the deviation's
            infer_rc = self.oracle.infer(b"".join(fr[:row]), self.rt)[0] or A.TFR_E_MALFORMED_PROTO
        over_64k = what.startswith("a 66 KiB")
        # 1. the first batch of a fresh decoder
        d = self.native.Decoder(self.sch, self.rt)
        try:
            b, _ = d.decode(data)
            self.check(b, want, f"first-batch decode: {msg}"); b.release()
            if over_64k:
                assert d.stats()["general_path_batches"] == 1, (tag, d.stats())
        finally:
            d.close()
        # 2. the steady state
        s0 = self.dec.stats()
        b = self.dec.submit(data)
        self.check(b, want, f"pipelined submit: {msg}"); b.release()
        s1 = self.dec.stats()
        if over_64k:
            assert s1["general_path_batches"] == s0["general_path_batches"] + 1, f"a 66 KiB record not on the general path: {s0} -> {s1}; {tag}"
        elif self.mode != "general" and cls in W.CANONICAL_CLASSES:
            if self.mode == "pipelined" and s1["speculative_redone"] != s0["speculative_redone"] \
                    and (s1["general_path_batches"] == s0["general_path_batches"] or self.bad_utf8):
                # a record larger than every slot learned so far is redone once (the tile kernel in the synchronising
                # decode, or the general kernels when the batch also holds malformed UTF-8, which only the pipelined
                # kernel transcodes); the same bytes again must then stay on the fast path
                b = self.dec.submit(data)
                self.check(b, want, f"pipelined submit, again: {msg}"); b.release()
                s0, s1 = s1, self.dec.stats()
            assert in_mode(self.mode, s0, s1), f"canonical record not decoded {self.mode}: {s0} -> {s1}; {tag}"
        elif self.mode == "general":
            assert in_mode("general", s0, s1), (tag, s0, s1)
        # 3. the general kernels only
        b, _ = self.gen_dec.decode(data)
        self.check(b, want, f"general kernels: {msg}"); b.release()
        # 4. inference over the same bytes
        rc, codes = self.oracle.infer(data, self.rt)
        rc = rc if infer_rc is None else infer_rc
        inf = self.native.Infer(self.rt)
        try:
            inf.update(data)
            got_rc, got = 0, inf.result()
        except self.native.TfrError as e:
            got_rc, got = e.code, None
        finally:
            inf.close()
        assert got_rc == rc, f"infer: status {got_rc} != oracle {rc}; {msg}"
        if rc == 0 and cls != "groups_25":
            assert got == codes, f"infer: {msg}"
        # back to the steady state: at once after a canonical record of a size the slots hold, after one relearning
        # batch otherwise (a non-canonical record can look like a shape change to the uniform kernel: relearned)
        relearn = cls not in W.CANONICAL_CLASSES or cls in ("multibyte", "many_entries")
        self.clean_submit(tag, not relearn)
        if relearn:
            self.clean_submit(tag, True)


ROWS = lambda n: [0, 31, 32, n // 2, n - 1]


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_wire_rewrites_match_the_oracle_on_every_path(native, oracle, cfg):
    h = Harness(native, oracle, cfg)
    R = random.Random(h.seed)
    rows = ROWS(h.n)
    k = 0
    try:
        # class A: every class at two rows, every extra-key kind once
        for cls in W.A_CLASSES:
            if cls == "seq" and h.rt == 0:
                continue
            for _ in range(2):
                r = rows[k % len(rows)]; k += 1
                p, what = W.rewrite(h.sch, h.rows[r], h.rt, cls, R, W=R.choice([12, 4]))
                h.run(cls, p, r, what)
        for variant in W.EXTRA_KEYS:
            r = rows[k % len(rows)]; k += 1
            p, what = W.rewrite(h.sch, h.rows[r], h.rt, "extra", R, variant=variant)
            h.run("extra", p, r, what)
        for d in DECOY_DISTANCES:
            r = rows[k % len(rows)]; k += 1
            p, what = W.rewrite(h.sch, h.rows[r], h.rt, "merge", R, variant=f"decoy_entry:{d}")
            h.run("merge", p, r, what)
        # class B: every error at a row of its own
        for cls in W.B_CLASSES:
            r = rows[k % len(rows)]; k += 1
            e = W.error_record(h.sch, h.rows[r], h.rt, cls, R)
            if e is None:
                continue
            p, code, field, what = e
            h.run(cls, p, r, what, code, field)
        for variant in sorted(W.MAL_SHAPES) + ["feature", "flist"]:
            r = rows[k % len(rows)]; k += 1
            e = W.error_record(h.sch, h.rows[r], h.rt, "malformed" if variant.startswith("mal_") else "bad_nesting", R, variant=variant)
            if e is None:
                continue
            p, code, field, what = e
            h.run("malformed" if variant.startswith("mal_") else "bad_nesting", p, r, what, code, field)
        # two errors in one batch (rows 31 and 32): the first row's; two in one record: the first field in schema order
        p1, c1, f1, w1 = W.error_record(h.sch, h.rows[31], h.rt, "kind_not_set", R)
        p2, _, _, w2 = W.error_record(h.sch, h.rows[32], h.rt, "malformed", R)
        h.run("two_rows", p1, 31, f"{w1}, then {w2} at row 32", c1, f1, more=[(32, p2)])
        two = W.two_errors_in_one_record(h.sch, h.rows[h.n - 1], h.rt, R)
        if two is not None:
            p, code, field, what = two
            h.run("two_fields", p, h.n - 1, what, code, field)
        # class C: damage inside one payload (canonical or rewritten), CRC recomputed
        for t in range(6):
            r = rows[k % len(rows)]; k += 1
            base = W.canonical(h.sch, h.rows[r], h.rt) if t % 2 else W.rewrite(h.sch, h.rows[r], h.rt, R.choice(W.A_CLASSES), R)[0]
            p, what = W.mutate(base, R)
            h.run("damage", p, r, what)
        st = h.dec.stats()
        print(f"{h.name}: {h.n} rows per batch, decoder stats {st}")
        if h.bad_utf8:
            assert st["transcode_reruns"] >= 1, st
    finally:
        h.close()
