"""TFR_F_RESYNC on the GPU: DROPMALFORMED and PERMISSIVE decoders (and tolerant schema inference) that resynchronise on the
next verified frame after a framing error.

The expectation of a block comes from the sequential walker (resync_walk.walk: its frames and lost regions) and the C
oracle's drop-mode decode of the kept frames (test_gpu_drop_malformed.expected, on the frames gathered back to back); the
failing records and the regions are then merged in entry order, and PERMISSIVE spreads the rows as test_gpu_permissive does."""
import os
import random
import struct

import numpy as np
import pytest

import resync_walk as RW
import test_gpu_drop_malformed as D
import test_gpu_permissive as PM
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200._cabi import HostColumn
from spark_tfrecord_b200.sqltypes import *  # noqa
from util import assert_columns_equal

pytestmark = pytest.mark.gpu

DROP = A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED | A.TFR_F_RESYNC
PERM = A.TFR_F_DEFAULT | A.TFR_F_PERMISSIVE | A.TFR_F_RESYNC


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


# ---------------------------------------------------------------------------------------------
# damage
# ---------------------------------------------------------------------------------------------
def header(length, crc_ok=True):
    h = struct.pack("<Q", length)
    c = pyref.masked_crc32c(h)
    return h + struct.pack("<I", c if crc_ok else c ^ 0x5A5A5A5A)


def flip_lencrc(fr, R_):
    fr = bytearray(fr)
    fr[8 + R_.randrange(4)] ^= 1 << R_.randrange(8)
    return bytes(fr)


def rewrite_len(fr, R_):
    """a different length with a recomputed header CRC: the chain follows it into the wrong place"""
    L = len(fr) - 16
    return header(max(0, L + R_.choice([-7, -3, 5, 11, 40]))) + fr[12:]


def oversize_len(fr, R_):
    return header((1 << 31) + R_.randrange(1 << 20)) + fr[12:]


def garbage(R_, kind, n):
    if kind == "zeros":
        return bytes(n)
    g = bytearray(R_.randbytes(n))
    if kind == "decoys":                        # header-valid frames whose payload CRC fails, and one with an oversize claim
        for _ in range(3):
            p = R_.randrange(max(1, n - 64))
            body = R_.randbytes(24)
            g[p:p + 40] = header(24) + body + struct.pack("<I", pyref.masked_crc32c(body) ^ 1)
        p = R_.randrange(max(1, n - 16))
        g[p:p + 12] = header(1 << 20)           # verifies, but runs past any block here: undecided on a non-final block
    return bytes(g[:n])


DAMAGE = ["lencrc", "rewrite_len", "oversize", "tail_truncated", "truncated_concat", "garbage_random", "garbage_zeros",
          "garbage_decoys", "every_record"]


def damage(kind, frames, seed):
    """the framed bytes of `frames` with damage of `kind` at a few seeded places"""
    R_ = random.Random(seed)
    fr = list(frames)
    n = len(fr)
    at = sorted(R_.sample(range(1, n - 1), 3))
    if kind == "lencrc":
        for i in at:
            fr[i] = flip_lencrc(fr[i], R_)
    elif kind == "rewrite_len":
        for i in at:
            fr[i] = rewrite_len(fr[i], R_)
    elif kind == "oversize":
        for i in at:
            fr[i] = oversize_len(fr[i], R_)
    elif kind == "tail_truncated":
        fr[-1] = fr[-1][:R_.randrange(13, len(fr[-1]) - 1)]
    elif kind == "truncated_concat":           # a part file cut off mid-record, then a good file
        fr[n // 2] = fr[n // 2][:R_.randrange(13, len(fr[n // 2]) - 1)]
    elif kind.startswith("garbage"):
        for i in at:
            fr[i] = garbage(R_, kind.split("_")[1], R_.randrange(1, 300)) + fr[i]
    elif kind == "every_record":
        fr = [flip_lencrc(f, R_) for f in fr]
    return b"".join(fr)


# ---------------------------------------------------------------------------------------------
# the expectation
# ---------------------------------------------------------------------------------------------
def expected(oracle, data, sch, rt, flags, is_final=True, cf=None) -> D.Expect:
    """walker entries + the oracle's drop-mode decode of the kept frames; PERMISSIVE (flags) with the corrupt-record column
    at cf (or None)"""
    data = bytes(data)
    entries, consumed = RW.walk(data, is_final)
    frames = [e for e in entries if e[0] == "frame"]
    kept = b"".join(data[a:b] for _, a, b in frames)
    perm = bool(flags & A.TFR_F_PERMISSIVE)
    sub = sch if cf is None else StructType([f for i, f in enumerate(sch.fields) if i != cf])
    e = D.expected(oracle, kept, sub, rt, A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED, True)
    assert not e.info["error_code"], e.info
    entry_of = [i for i, x in enumerate(entries) if x[0] == "frame"]     # frame index -> entry index
    spans = []                                                          # (entry, offset, nbytes, code, field)
    for i, _, code, f in e.dropped:
        _, a, b = frames[i]
        spans.append((entry_of[i], a, b - a, code, f + (cf is not None and f >= cf)))
    for k, x in enumerate(entries):
        if x[0] == "region":
            spans.append((k, x[1], x[2] - x[1], x[3], -1))
    spans.sort()
    info = {"n_rows": e.info["n_rows"], "n_records": len(entries), "consumed_bytes": consumed, "error_code": 0,
            "error_row": -1, "error_field": -1}
    cols = e.columns
    if perm:
        bad = [s[0] for s in spans]
        n_total = e.info["n_rows"] + len(bad)
        cols = [PM.expand(c, bad, n_total) for c in cols]
        if cf is not None:
            cols.insert(cf, corrupt_column(data, entries, spans, n_total))
        info["n_rows"] = n_total
    exp = D.Expect(cols, info, [(r, o, c, f) for r, o, _, c, f in spans])
    exp.spans = spans
    return exp


def corrupt_column(data, entries, spans, n_total):
    """a failing frame's payload, a lost region's bytes as they are"""
    bad = [s[0] for s in spans]
    parts = []
    for r, o, nb, _, _ in spans:
        parts.append(data[o:o + nb] if entries[r][0] == "region" else data[o + 12:o + nb - 4])
    bits = np.zeros(n_total, np.uint8)
    bits[bad] = 1
    cum = np.concatenate([[0], np.cumsum([len(p) for p in parts], dtype=np.int64)]).astype(np.int32)
    bb = np.searchsorted(np.asarray(bad, np.int64), np.arange(n_total + 1), side="left")
    vals = np.frombuffer(b"".join(parts), np.uint8) if parts else np.zeros(0, np.uint8)
    return HostColumn(TFR_T_BINARY, 0, n_total, np.packbits(bits, bitorder="little"), [cum[bb]], vals)


def check_batch(b, sch, exp, what, rows=True):
    D.check_info(b, exp, what)
    assert b.dropped_spans() == exp.spans, f"{what}: spans {b.dropped_spans()} != {exp.spans}"
    assert_columns_equal(b.to_host(), exp.columns, None, what)
    if rows:
        D.check_rows(b, sch, exp, None, what)


def regions_of(exp):
    return [s for s in exp.spans if s[3] in A.FRAMING_ERRORS]


def decoder(native, sch, rt, flags, pos):
    full, cf = PM.with_corrupt(sch, pos) if flags & A.TFR_F_PERMISSIVE else (sch, None)
    return full, cf, native.Decoder(full, rt, flags=flags, corrupt_field=cf)


MODES = [("drop", DROP, None), ("perm", PERM, "middle"), ("perm_nocol", PERM, None)]
CORPORA = ["cfg2", "sequence_example", "byte_array"]


def corpus(name, n, seed):
    return D.CORPORA[name](n, seed)


# ---------------------------------------------------------------------------------------------
# 1. fresh decoders: every damage kind, both modes
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", DAMAGE)
@pytest.mark.parametrize("name", CORPORA)
@pytest.mark.parametrize("mode, flags, pos", MODES, ids=[m[0] for m in MODES])
def test_fresh(native, oracle, name, kind, mode, flags, pos):
    if name == "byte_array" and flags & A.TFR_F_PERMISSIVE:
        pytest.skip("PERMISSIVE takes no ByteArray records")
    sch, rt, rows, frames = corpus(name, 300, 11 + len(kind))
    data = damage(kind, frames, 5 + len(kind) + len(name))
    full, cf, dec = decoder(native, sch, rt, flags, pos)
    exp = expected(oracle, data, full, rt, flags, True, cf)
    assert exp.spans and (regions_of(exp) or kind == "truncated_concat"), (kind, exp.spans[:4])
    what = f"{name}/{kind}/{mode}"
    b, used = dec.decode(data)
    assert used == exp.info["consumed_bytes"] == len(data), what
    check_batch(b, full, exp, what)
    st = dec.stats()
    reg = regions_of(exp)
    assert st["lost_regions"] == len(reg) and st["lost_region_bytes"] == sum(s[2] for s in reg), (what, st)
    recs = len(exp.spans) - len(reg)
    assert st["records_corrupt" if flags & A.TFR_F_PERMISSIVE else "records_dropped"] == recs, (what, st)
    b.release()
    b, _ = dec.decode(data)                                   # (a batch's rows are built once: the partitioned ones need another)
    D.check_rows(b, full, exp, D.PART, what + " partitioned")
    b.release()
    dec.close()


def test_truncated_concat_swallows_then_resyncs(native, oracle):
    """rule 6: a record cut off and followed by a good file keeps its claimed length (its header verifies), swallowing the
    records that lie inside it; it fails its payload CRC (a record error) or runs past the block (a region); either way the
    frames after it are read"""
    sch, rt, rows, frames = corpus("cfg2", 200, 3)
    cut = frames[50][:len(frames[50]) // 2]
    data = b"".join(frames[:50]) + cut + b"".join(frames)
    exp = expected(oracle, data, sch, rt, DROP)
    dec = native.Decoder(sch, rt, flags=DROP)
    b, used = dec.decode(data)
    check_batch(b, sch, exp, "truncated + concatenated")
    assert 50 + 150 <= b.n_rows < 250, b.n_rows            # some of the second file's records are swallowed, not all
    b.release()
    dec.close()


# ---------------------------------------------------------------------------------------------
# 2. the pipelined steady state: clean blocks between damaged ones
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode, flags, pos", MODES[:2], ids=[m[0] for m in MODES[:2]])
@pytest.mark.parametrize("name", ["cfg2", "byte_array"])
def test_pipelined(native, oracle, name, mode, flags, pos):
    if name == "byte_array" and flags & A.TFR_F_PERMISSIVE:
        pytest.skip("PERMISSIVE takes no ByteArray records")
    sch, rt, rows, frames = corpus(name, 1500, 21)
    clean = b"".join(frames)
    full, cf, dec = decoder(native, sch, rt, flags, pos)
    want_clean = expected(oracle, clean, full, rt, flags, True, cf)
    for _ in range(3):
        dec.submit(clean).release()
    for k, kind in enumerate(["lencrc", "garbage_decoys", "oversize", "tail_truncated"]):
        s0 = dec.stats()
        b = dec.submit(clean)
        b.unsafe_rows_async(True)
        check_batch(b, full, want_clean, f"{name} clean {k}")
        b.release()
        d = D.delta(s0, dec.stats())
        assert d["speculative_submits"] == 1 and d["speculative_redone"] == 0 and d["lost_regions"] == 0, d
        data = damage(kind, frames, 40 + k)
        exp = expected(oracle, data, full, rt, flags, True, cf)
        s0 = dec.stats()
        b = dec.submit(data)
        b.unsafe_rows_async(True)
        assert b.consumed() == exp.info["consumed_bytes"]
        check_batch(b, full, exp, f"{name} {kind}")
        b.release()
        d = D.delta(s0, dec.stats())
        assert d["speculative_submits"] == 1 and d["speculative_redone"] == 1, d
        assert d["lost_regions"] == len(regions_of(exp)), d
    dec.close()


# ---------------------------------------------------------------------------------------------
# 3. streamed in blocks: every streamed result equals the single-block one
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lencrc", "garbage_decoys", "truncated_concat", "rewrite_len"])
@pytest.mark.parametrize("mode, flags, pos", MODES[:2], ids=[m[0] for m in MODES[:2]])
def test_streamed(native, oracle, kind, mode, flags, pos):
    sch, rt, rows, frames = corpus("cfg2", 400, 9)
    data = damage(kind, frames, 77 + len(kind))
    full, cf, dec = decoder(native, sch, rt, flags, pos)
    whole = expected(oracle, data, full, rt, flags, True, cf)
    want_spans = [(o, nb, c) for _, o, nb, c, _ in whole.spans]
    for block in (4096, 9001, 65536):
        pos_, spans, n_rows = 0, [], 0
        size = block
        while True:
            chunk = data[pos_:pos_ + size]
            final = pos_ + len(chunk) >= len(data)
            exp = expected(oracle, chunk, full, rt, flags, final, cf)
            b = dec.submit(chunk, is_final=final)
            used = b.consumed()
            assert used == exp.info["consumed_bytes"], (block, pos_, used, exp.info)
            check_batch(b, full, exp, f"{kind} block {block} at {pos_}", rows=False)
            spans += [(pos_ + o, nb, c) for _, o, nb, c, _ in b.dropped_spans()]
            n_rows += b.n_rows
            b.release()
            if final:
                break
            if used == 0:                      # an unresolved region (or a large record): the same start, more bytes
                size += block
                continue
            pos_ += used
            size = block
        assert spans == want_spans, (block, spans[:5], want_spans[:5])
        assert n_rows == whole.info["n_rows"], block
    dec.close()


# ---------------------------------------------------------------------------------------------
# 4. the reader and schema inference
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gz", [False, True], ids=["plain", "gz"])
def test_default_source_load(native, oracle, tmp_path, gz):
    import gzip
    from spark_tfrecord_b200 import io as tio
    sch, rt, rows, frames = corpus("cfg2", 300, 4)
    data = damage("garbage_decoys", frames, 8)
    path = str(tmp_path / ("part.tfrecord" + (".gz" if gz else "")))
    with (gzip.open if gz else open)(path, "wb") as f:
        f.write(data)
    entries, _ = RW.walk(data, True)
    kept = str(tmp_path / "kept.tfrecord")
    with open(kept, "wb") as f:                                # the frames the walker keeps, as a file of their own
        f.write(b"".join(data[e[1]:e[2]] for e in entries if e[0] == "frame"))
    got = tio.DefaultSource().load(path, sch, {"mode": "DROPMALFORMED", "resyncFraming": "true"})
    assert got == tio.DefaultSource().load(kept, sch, {"mode": "DROPMALFORMED"})
    assert len(got) == 300                                   # the garbage went in front of records: every record is read
    with pytest.raises(native.TfrError):                     # without the option the framing error still fails the file
        tio.DefaultSource().load(path, sch, {"mode": "DROPMALFORMED"})
    inferred = tio.DefaultSource().inferSchema({"mode": "DROPMALFORMED", "resyncFraming": "true"}, [path])
    names = {f.name for f in inferred.fields}
    assert names == {f.name for f in sch.fields}, names


def result_or_error(native, inf):
    """the merged names, or the error merging them raises (a corpus can hold conflicting types)"""
    try:
        return inf.result()
    except native.TfrError as e:
        return type(e), e.code


@pytest.mark.parametrize("kind", ["lencrc", "garbage_decoys", "tail_truncated", "every_record"])
@pytest.mark.parametrize("mode", ["DROPMALFORMED", "PERMISSIVE"])
def test_inference(native, oracle, kind, mode):
    sch, rt, rows, frames = corpus("sequence_example" if kind == "lencrc" else "cfg2", 200, 13)
    data = damage(kind, frames, 3 + len(kind))
    entries, consumed = RW.walk(data, True)
    kept = b"".join(data[e[1]:e[2]] for e in entries if e[0] == "frame")
    flags = (A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED) if mode == "DROPMALFORMED" else (A.TFR_F_DEFAULT | A.TFR_F_PERMISSIVE)
    name = "_corrupt_record" if mode == "PERMISSIVE" else None
    ref = native.Infer(rt, 0, flags, name)
    if kept:
        ref.update(kept)
    want_skipped = ref.skipped()
    want = result_or_error(native, ref)
    ref.close()
    inf = native.Infer(rt, 0, flags | A.TFR_F_RESYNC, name)
    assert inf.update_block(data, True) == consumed == len(data)
    got_skipped = inf.skipped()
    assert result_or_error(native, inf) == want
    frames_ = [e for e in entries if e[0] == "frame"]
    entry_of = [i for i, e in enumerate(entries) if e[0] == "frame"]
    exp = sorted([(entry_of[i], frames_[i][1], c, -1) for i, _, c, _ in want_skipped] +
                 [(k, e[1], e[3], -1) for k, e in enumerate(entries) if e[0] == "region"])
    assert got_skipped == exp, (got_skipped[:4], exp[:4])
    inf.close()


# ---------------------------------------------------------------------------------------------
# 5. the flag is opt-in
# ---------------------------------------------------------------------------------------------
def test_without_the_flag_framing_still_ends_the_block(native, oracle):
    sch, rt, rows, frames = corpus("cfg2", 200, 6)
    data = damage("lencrc", frames, 2)
    dec = native.Decoder(sch, rt, flags=A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED)
    b, used = dec.decode(data)
    assert b.info["error_code"] == A.TFR_E_CRC_LENGTH and used < len(data)
    assert dec.stats()["lost_regions"] == 0
    b.release()
    dec.close()
