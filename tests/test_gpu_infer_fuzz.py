"""Schema inference on the GPU (tfr_infer_*, infer.cuh) against the oracle over tests/infer_corpus.py's seeded corpora.

Every batch is inferred three ways, and each must give the oracle's status and, when that is 0, its {name: code} map:
  * `Infer.update` with the bytes in host memory, and with a device tensor at an odd address;
  * `Infer.update_block` over the same bytes in random blocks: tiny ones, ends inside a frame header and inside a
    payload, then `is_final`; each block's consumed count must be the end of its last whole frame;
  * several `update` calls, one per "file": the merged result is the oracle's over the concatenation, including the
    UNSUPPORTED_TYPE of a name of all-empty steps (ArrayType(ArrayType(null))) that another file types, at `result()`.
The oracle's inference reads frames without verifying CRCs; the GPU verifies them as the reference's record reader
does.  A batch with a flipped data CRC must therefore fail with the error of the first failing record before it, or
with TFR_E_CRC_DATA.
Fixed cases: the six regressions of infer_corpus.payload_table(); 200 k records of about 5,000 names in a grid-filling
launch; the two names of equal 64-bit hash in records of different warps; the exact limits (1,024 entries in one map,
65,536 distinct names in one call); a record over a limit after a failing record (the failing record's error wins)."""
import random

import numpy as np
import pytest

import infer_corpus as C
from oracle import pyref
from oracle.pyref import ld, map_entry
from spark_tfrecord_b200 import _cabi as A

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def _infer(native, rt, feed):
    """-> (status, names -> codes or None): `feed(inf)` makes the update calls"""
    inf = native.Infer(rt)
    try:
        feed(inf)
        return 0, inf.result()
    except native.TfrError as e:
        return e.code, None
    finally:
        inf.close()


def _on_device_odd(data: bytes):
    import torch
    buf = torch.empty(len(data) + 1, dtype=torch.uint8, device="cuda")
    t = buf[1:]
    t.copy_(torch.frombuffer(bytearray(data), dtype=torch.uint8))
    return t


def _blocks(inf, b: C.Batch, R: random.Random):
    """update_block over random blocks; every consumed count is the end of the block's last whole frame"""
    data, ends = b.data, b.frame_ends
    starts = [0] + ends[:-1]
    pos = 0
    while True:
        cut = R.choice(["tiny", "header", "payload", "big"])
        nxt = [e for e in ends if e > pos]
        if cut == "tiny":
            end = pos + R.randrange(1, 40)
        elif cut == "header" and nxt:
            s = starts[ends.index(nxt[0])]
            end = max(pos + 1, s + R.randrange(1, 12))               # inside the next frame's header
        elif cut == "payload" and nxt:
            k = R.randrange(len(nxt))
            end = nxt[k] - R.randrange(1, 5) if nxt[k] - pos > 4 else nxt[k]
        else:
            end = pos + R.randrange(1, 1 << 16)
        end = min(end, len(data))
        final = end == len(data)
        used = inf.update_block(data[pos:end], final)
        whole = [e for e in ends if pos < e <= end]
        want = (whole[-1] - pos) if whole else 0
        if final:
            want = len(data) - pos if not b.truncated else want
        assert used == want, f"consumed {used} != {want} (block {pos}..{end} of {len(data)})"
        pos += used
        if final:
            return


def _want(oracle, b: C.Batch):
    """the oracle's (status, names -> codes) for the batch as the GPU must see it"""
    if b.crc_row is not None:
        rc, codes = oracle.infer(b.data[:b.frame_ends[b.crc_row] - len(pyref.frame_fast(b.payloads[b.crc_row]))], b.rt)
        return (rc or A.TFR_E_CRC_DATA), None
    rc, codes = oracle.infer(b.data, b.rt)
    return rc, (codes if rc == 0 else None)


def _check(native, oracle, b: C.Batch, R: random.Random, what: str):
    want = _want(oracle, b)
    msg = f"{what}: {b.describe()}"
    got = _infer(native, b.rt, lambda inf: inf.update(np.frombuffer(b.data, np.uint8)))
    assert got == want, f"update (host): {got} != {want}; {msg}"
    got = _infer(native, b.rt, lambda inf: inf.update(_on_device_odd(b.data)))
    assert got == want, f"update (device, odd address): {got} != {want}; {msg}"
    got = _infer(native, b.rt, lambda inf: _blocks(inf, b, R))
    assert got == want, f"update_block: {got} != {want}; {msg}"
    return want


@pytest.mark.parametrize("rt", [0, 1])
def test_seeded_batches_match_the_oracle(native, oracle, rt):
    R = random.Random(rt)
    seen = {}
    for seed in range(48):
        n = R.choice([1, 2, 33, 64, 200])
        b = C.batch(seed, rt, n)
        rc, _ = _check(native, oracle, b, R, f"seed {seed}")
        seen[rc] = seen.get(rc, 0) + 1
    # the corpus reaches every verdict it is built for
    want = {0, A.TFR_E_KIND_MISMATCH, A.TFR_E_MALFORMED_PROTO, A.TFR_E_TRUNCATED, A.TFR_E_CRC_DATA}
    if rt == 1:
        want |= {A.TFR_E_UNSUPPORTED_TYPE}
    assert want <= set(seen), seen


@pytest.mark.parametrize("rt", [0, 1])
def test_files_merge_like_one_concatenation(native, oracle, rt):
    """one update per file; names merge across files, and a code-10 conflict between files surfaces at result()"""
    R = random.Random(100 + rt)
    for seed in range(12):
        files = [C.batch(1000 * seed + k, rt, R.choice([1, 20, 90]), mode="clean") for k in range(R.randrange(2, 5))]
        if rt == 1 and seed % 3 == 0:
            key = C.EMPTY_STEPS[0]
            files[0].payloads.append(ld(2, map_entry(key, C.fl(C.i64(), C.f32()))))
            files[-1].payloads.append(ld(2, map_entry(key, C.fl(C.byt(b"q")))))
        datas = [b"".join(pyref.frame_fast(p) for p in f.payloads) for f in files]
        want = oracle.infer(b"".join(datas), rt)
        want = (want[0], want[1] if want[0] == 0 else None)
        got = _infer(native, rt, lambda inf: [inf.update(np.frombuffer(d, np.uint8)) for d in datas])
        assert got == want, f"seed {seed}, {len(files)} files: {got} != {want}"
        if rt == 1 and seed % 3 == 0:
            assert want[0] == A.TFR_E_UNSUPPORTED_TYPE


@pytest.mark.parametrize("name,payload,rt,rc,codes", C.payload_table(), ids=[t[0] for t in C.payload_table()])
def test_regressions(native, oracle, name, payload, rt, rc, codes):
    data = pyref.frame(payload)
    assert oracle.infer(data, rt) == (rc, codes) if rc == 0 else oracle.infer(data, rt)[0] == rc
    b = C.Batch(rt, [payload], [])
    _check(native, oracle, b, random.Random(name), name)
    # the same record among clean ones, at a row of the second warp of a CTA and at a later CTA
    for row in (1, 37):
        clean = C.batch(7, rt, 64, mode="clean").payloads
        clean[row] = payload
        _check(native, oracle, C.Batch(rt, clean, [(row, name)]), random.Random(row), f"{name} at row {row}")


def test_equal_hash_names_in_different_warps(native, oracle):
    for rows in ((0, 1), (0, 2), (5, 4000)):
        ps = [ld(1, map_entry(b"k%d" % i, C.i64(i))) for i in range(max(rows) + 1)]
        ps[rows[0]] = ld(1, map_entry(C.COLL_A, C.i64(1)))
        ps[rows[1]] = ld(1, map_entry(C.COLL_B, C.f32(1.0, 2.0)))
        b = C.Batch(0, ps, [(rows[0], "A"), (rows[1], "B")])
        rc, codes = _check(native, oracle, b, random.Random(rows[1]), f"A at row {rows[0]}, B at row {rows[1]}")
        assert rc == 0 and codes[C.COLL_A] == 1 and codes[C.COLL_B] == 5


def test_many_warps_insert_the_same_names(native, oracle):
    """200 k records over ~5,000 names: far more records than the sm_count x 16 CTAs of two warps, so every slot of
    the table is inserted into and atomicMax'ed by many warps at once"""
    R = random.Random(5)
    names = C.names_pool(R, 5000)
    rng = np.random.default_rng(5)
    feats = [C.i64(1), C.i64(1, 2), C.f32(1.0), C.byt(b"a"), C.i64(), C.f32(1.0, 2.0, 3.0), C.byt(b"a", b"b")]
    pick = rng.integers(0, len(names), (200_000, 4))
    kind = rng.integers(0, len(feats), (200_000, 4))
    ps = [ld(1, b"".join(map_entry(names[pick[r, k]], feats[kind[r, k]]) for k in range(4))) for r in range(200_000)]
    b = C.Batch(0, ps, [])
    want = _want(oracle, b)
    assert want[0] == 0 and len(want[1]) > 4900
    got = _infer(native, 0, lambda inf: inf.update(np.frombuffer(b.data, np.uint8)))
    assert got == want
    got = _infer(native, 0, lambda inf: inf.update(_on_device_odd(b.data)))
    assert got == want


def _wide(n, key=b"k"):
    return ld(1, b"".join(map_entry(key + b"%05d" % i, C.i64(i)) for i in range(n)))


def test_entry_limit_is_exact(native, oracle):
    for rt in (0, 1):
        for n, ok in ((1024, True), (1025, False)):
            p = _wide(n)
            if rt == 1:
                p += ld(2, map_entry(b"s", C.fl(C.i64(1))))
            rc, codes = _infer(native, rt, lambda inf: inf.update(pyref.frame_fast(p)))
            if ok:
                assert (rc, codes) == oracle.infer(pyref.frame_fast(p), rt) and len(codes) == n + rt
            else:
                assert rc == A.TFR_E_BATCH_TOO_LARGE
    # the same limit in feature_lists
    p = ld(2, b"".join(map_entry(b"s%05d" % i, C.fl(C.i64(i))) for i in range(1025)))
    assert _infer(native, 1, lambda inf: inf.update(pyref.frame_fast(p)))[0] == A.TFR_E_BATCH_TOO_LARGE


def test_name_limit_is_exact(native):
    for n, ok in ((65536, True), (65537, False)):
        names = [b"n%06d" % i for i in range(n)]
        ps = [ld(1, b"".join(map_entry(k, C.i64(1)) for k in names[i:i + 64])) for i in range(0, n, 64)]
        rc, codes = _infer(native, 0, lambda inf: inf.update(b"".join(pyref.frame_fast(p) for p in ps)))
        if ok:
            assert rc == 0 and codes == {k: 1 for k in names}
        else:
            assert rc == A.TFR_E_BATCH_TOO_LARGE


def test_an_earlier_failing_record_wins_over_a_limit(native, oracle):
    clean = C.batch(11, 0, 40, mode="clean").payloads
    bad = ld(1, map_entry(b"k", C.UNSET))
    for err_row, lim_row in ((3, 10), (0, 39), (10, 3)):
        ps = list(clean)
        ps[err_row], ps[lim_row] = bad, _wide(1025)
        data = b"".join(pyref.frame_fast(p) for p in ps)
        rc, _ = _infer(native, 0, lambda inf: inf.update(data))
        if err_row < lim_row:
            assert rc == oracle.infer(data, 0)[0] == A.TFR_E_KIND_MISMATCH, (err_row, lim_row)
        else:
            assert rc == A.TFR_E_BATCH_TOO_LARGE, (err_row, lim_row)
    # a full name table: the record's error is the reference's answer (it has no table)
    names = [ld(1, b"".join(map_entry(b"n%06d" % (i + k), C.i64(1)) for k in range(64))) for i in range(0, 66048, 64)]
    names[700] = bad                                      # 65,984 names are left
    data = b"".join(pyref.frame_fast(p) for p in names)
    assert _infer(native, 0, lambda inf: inf.update(data))[0] == A.TFR_E_KIND_MISMATCH
