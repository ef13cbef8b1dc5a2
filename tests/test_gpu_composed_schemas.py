"""GPU tests of schemas that combine every lowering -- dense and sparse vectors, ragged fields (row lengths and row splits),
extendedTypes=true fields, the generated fields and the corrupt-record column -- against tests/composed_rows.py, on every
decode path, in every mode and through every view.  Every case names the path it means and checks it through the
decoder's or encoder's counters: a right answer from the wrong path fails.

Paths: general (TFR_DISABLE_FAST), tile 4 + 1 (records up to 625 B), tile 12 + 3 (a larger record in the batch), the
packed tile of a pipelined submit (one record of 2.5 KB among ones of a few hundred bytes), the large-record kernel, and the pipelined
steady state.  Boundaries: 64 / 65 and 128 / 129 narrowed columns (narrow_kernel and widen_kernel take 64 per launch), and
127 / 128 / 129 lowered fields (the fast paths take at most 128, sparse and ragged parts included).

No counter tells the two tile kernels apart (both count as a count-mode batch): the 4 + 1 and 12 + 3 cases pick their
records' sizes for the geometry (at most 600 B, and one record of 160 eight-byte longs), and the counters show that a tile
kernel ran.  The encoders count only their pipelined submits' general emits."""
import ctypes as C
import os

import numpy as np
import pytest

import composed_rows as CR
import int64_types as I
import position_walk as PW
import ragged_rows as RR
import resync_walk as RW
import test_gpu_batch_outputs as BO
import test_gpu_row_index as RI
import vector_rows as V
from oracle import pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

pytestmark = pytest.mark.gpu

VERIFY = A.TFR_F_VERIFY_CRC
MODES = {"failfast": (VERIFY, PW.FAILFAST, False),
         "drop": (VERIFY | A.TFR_F_DROP_MALFORMED, PW.DROPMALFORMED, False),
         "permissive": (VERIFY | A.TFR_F_PERMISSIVE, PW.PERMISSIVE, False),
         "permissive_resync": (VERIFY | A.TFR_F_PERMISSIVE | A.TFR_F_RESYNC, PW.PERMISSIVE, True)}


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def delta(s0, s1):
    return {k: s1[k] - s0[k] for k in s0}


def decoder(native, sch, opts, flags=VERIFY, general=False):
    """a decoder of `sch`; with a corrupt-record column in `opts`, a PERMISSIVE one"""
    kw = dict(flags=flags, **opts.native())
    if opts.corrupt is not None:
        kw["corrupt_field"] = opts.corrupt
        kw["flags"] = flags | A.TFR_F_PERMISSIVE
    if not general:
        return native.Decoder(sch, 0, **kw)
    os.environ["TFR_DISABLE_FAST"] = "1"
    try:
        return native.Decoder(sch, 0, **kw)
    finally:
        del os.environ["TFR_DISABLE_FAST"]


def want_columns(sch, opts, rows):
    return [CR.canon(list(CR.column_row(sch, r, opts))) for r in rows]


def check_batch(b, sch, opts, exp, what):
    info = b.info
    got_err = (info["error_code"], info["error_row"], info["error_field"]) if info["error_code"] else None
    assert got_err == exp.error, (what, got_err, exp.error)
    assert [(d[0], d[2], d[3]) for d in b.dropped()] == exp.dropped, (what, b.dropped(), exp.dropped)
    assert b.n_rows == len(exp.rows), (what, b.n_rows, len(exp.rows))
    got = CR.columns_rows(b.to_host(), b.n_rows)
    want = want_columns(sch, opts, exp.rows)
    for r, (g, w) in enumerate(zip(got, want)):
        assert g == w, (what, r, [(i, x, y) for i, (x, y) in enumerate(zip(g, w)) if x != y][:3])


def on_path(d, path, what):
    if path == "general":
        assert d["general_path_batches"] == 1 and d["large_record_batches"] == 0, (what, d)
    elif path == "large":
        assert d["large_record_batches"] == 1 and d["general_path_batches"] == 0, (what, d)
    else:                                                   # a tile kernel: counted as a count-mode batch
        assert d["count_mode_batches"] == 1 and d["general_path_batches"] == 0 and d["large_record_batches"] == 0, (what, d)


def _pad_field(sch, seed):
    """the schema with a nullable ArrayType(LongType) `pad` at a seeded place: a plain depth-1 leaf whose length sets the
    record sizes each path needs"""
    r = np.random.default_rng(seed + 7)
    fields = list(sch.fields)
    fields.insert(int(r.integers(0, len(fields) + 1)), StructField("pad", ArrayType(LongType()), True))
    return StructType(fields)


def _with_pad(sch, rows, sizes):
    """rows with `pad` set to sizes[k] longs (None: null)"""
    p = sch.names.index("pad")
    out = []
    for k, r in enumerate(rows):
        n = sizes[k] if k < len(sizes) else None
        r = list(r)
        r[p] = None if n is None else [(k * 7919 + j) * 1_000_003 for j in range(n)]
        out.append(tuple(r))
    return out


# ---------------------------------------------------------------------------------------------
# a. seeded composed schemas on every decode path
# ---------------------------------------------------------------------------------------------
PATHS = ["general", "tile_4_1", "tile_12_3", "packed", "large", "pipelined"]
SEEDS = range(24)


def seeded_case(seed, n_fields):
    """(writer schema, decoder schema, opts) of a seed: every lowering on, and a vector, a ragged field and an extendedTypes
    field at seeded places among the drawn ones; the generated fields at seeded places.  Over the seeds k * 6 + p (p: the
    path) the options run through (dense, row lengths), (sparse, row splits), and with a corrupt-record column at a seeded
    place (a PERMISSIVE decoder) (dense, row splits), (sparse, row lengths)."""
    k = seed // 6
    fmt, splits, corrupt = ("dense", "sparse")[k % 2], (k + k // 2) % 2 == 1, k >= 2
    opts = CR.Opts(fmt, True, splits, True)
    ws = CR.with_kinds(CR.seeded_schema(seed, n_fields, opts), seed, [("v", "vector"), ("x", "long:2"), ("e", "short:1")])
    ws = _pad_field(ws, seed)
    ds, cidx = CR.with_extras(ws, seed, corrupt)
    assert any(isinstance(f.dataType, VectorUDT) for f in ws) and RR.ragged_fields(ws)
    assert any(I.leaf_id(f.dataType) for f in ws)
    return ws, ds, CR.Opts(fmt, True, splits, True, cidx)


@pytest.mark.parametrize("seed", SEEDS)
def test_seeded_schema_on_its_path(native, seed):
    path = PATHS[seed % len(PATHS)]
    ws, ds, opts = seeded_case(seed, 10 if path == "tile_4_1" else 18)
    what = f"seed {seed} {path} {opts}"
    n = {"general": 200, "tile_4_1": 200, "tile_12_3": 200, "packed": 96, "large": 24, "pipelined": 3000}[path]
    rows = CR.seeded_rows(ws, opts, n, seed)
    if path == "tile_4_1":                                  # every payload within the 4 + 1 tile's 625 bytes
        rows = [r for r in _with_pad(ws, rows, []) if len(CR.encode(ws, [r], opts)) - 16 <= 600][:120]
        assert len(rows) > 60, what
    sizes = {"tile_12_3": [3] * 50 + [160], "large": [12_000] * 8, "packed": [3] * 31 + [400]}.get(path, [])
    rows = _with_pad(ws, rows, sizes)
    data = CR.encode(ws, rows, opts)
    if path == "tile_12_3":
        assert max(e[2] - e[1] - 16 for e in RW.chain(data, 0, True)[0]) > 625, what
    exp = CR.Expect(ds, opts, data, PW.FAILFAST if opts.corrupt is None else PW.PERMISSIVE)
    assert exp.error is None and len(exp.rows) == len(rows)
    buf = np.frombuffer(data, dtype=np.uint8)
    dec = decoder(native, ds, opts, general=path == "general")
    try:
        if path in ("packed", "pipelined"):
            learn = data
            if path == "packed":                            # the same sizes, the large record at another row
                learn = CR.encode(ws, _with_pad(ws, rows, [3] * 40 + [400]), opts)
            s0 = dec.stats()
            b, _ = dec.decode(np.frombuffer(learn, dtype=np.uint8))
            assert b.info["error_code"] == 0, (what, b.info)
            b.release()
            on_path(delta(s0, dec.stats()), "tile", f"{what}: the learning decode")      # (shapes are learned on a tile)
            for k in range(2):
                b = dec.submit(np.frombuffer(learn, dtype=np.uint8))
                assert b.info["error_code"] == 0, (what, b.info)
                b.release()
            for k in range(2):
                s0 = dec.stats()
                b = dec.submit(buf)
                check_batch(b, ds, opts, exp, f"{what} steady submit {k}")
                b.release()
                d = delta(s0, dec.stats())
                assert d["speculative_submits"] == 1 and d["speculative_redone"] == 0, (what, d)
                assert d["general_path_batches"] == 0 and d["large_record_batches"] == 0, (what, d)
        else:
            s0 = dec.stats()
            b, used = dec.decode(buf)
            assert used == len(data)
            check_batch(b, ds, opts, exp, what)
            b.release()
            on_path(delta(s0, dec.stats()), "large" if path == "large" else path, what)
    finally:
        dec.close()


# the fast paths hand a batch whose ragged parts disagree to the general path
@pytest.mark.parametrize("path", ["tile", "large"])
@pytest.mark.parametrize("splits", [False, True])
def test_ragged_mismatch_goes_to_the_general_path(native, path, splits):
    seed = 31 + splits
    opts = CR.Opts("sparse", True, splits, True)
    ws = _pad_field(CR.seeded_schema(seed, 14, opts, ["vector", "long:2", "short:2", "string:2", "date:1", "int:0"]), seed)
    rows = CR.seeded_rows(ws, opts, 60 if path == "tile" else 24, seed)
    rows = _with_pad(ws, rows, [12_000] * 8 if path == "large" else [])
    low = CR.lowered_schema(ws, opts)
    rg = [i for i, f in enumerate(ws) if isinstance(f.dataType, ArrayType) and isinstance(f.dataType.elementType, ArrayType)]
    bad_at, x = len(rows) // 2, rg[-1]
    lr = list(CR.lower_row(ws, rows[bad_at], opts))
    lr[len(low) - 1] = [1] if splits else [-1]              # x's part: splits that do not start at 0; a negative length
    payloads = [pyref.frame(pyref.serialize_example_bytes(low, CR.lower_row(ws, r, opts))) for r in rows]
    payloads[bad_at] = pyref.frame(pyref.serialize_example_bytes(low, tuple(lr)))
    data = b"".join(payloads)
    exp = CR.Expect(ws, opts, data, PW.FAILFAST)
    assert exp.error == (A.TFR_E_BAD_NESTING, bad_at, x)
    clean = CR.encode(ws, rows, opts)
    dec = decoder(native, ws, opts)
    try:
        s0 = dec.stats()
        b, _ = dec.decode(np.frombuffer(clean, dtype=np.uint8))
        check_batch(b, ws, opts, CR.Expect(ws, opts, clean, PW.FAILFAST), "clean")
        b.release()
        on_path(delta(s0, dec.stats()), path, "clean")
        s0 = dec.stats()
        b, _ = dec.decode(np.frombuffer(data, dtype=np.uint8))
        check_batch(b, ws, opts, exp, "mismatch")
        b.release()
        d = delta(s0, dec.stats())
        assert d["general_path_batches"] == 1, d
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# c. modes: one batch with one of each damage
# ---------------------------------------------------------------------------------------------
def damaged_case(seed, corrupt):
    """a composed schema with a sparse vector, a ragged field and an extendedTypes field among seeded ones, and a batch of
    24 records: a CRC flip at 3, a malformed sparse part at 7, a row-lengths / row-splits part of the wrong kind at 11 and
    one that disagrees with its values at 13, a kind mismatch on the extendedTypes field at 15, a damaged frame header at
    19"""
    splits = seed % 2 == 1
    opts = CR.Opts("sparse", True, splits, True)
    base = CR.seeded_schema(seed, 12, opts)
    r = np.random.default_rng(seed)
    fields = list(base.fields)
    for nm, kind in (("v", "vector"), ("x", "int:2"), ("e", "byte:1")):
        fields.insert(int(r.integers(0, len(fields) + 1)), CR.make_field(nm, kind, True))
    ws = StructType(fields)
    rows = CR.seeded_rows(ws, opts, 24, seed)
    low = CR.lowered_schema(ws, opts)
    names = low.names

    def payload(k, patch=None):
        lr = list(CR.lower_row(ws, rows[k], opts))
        sch = low
        if patch:
            fs = list(low.fields)
            for nm, (dt, val) in patch.items():
                j = names.index(nm)
                fs[j] = StructField(nm, dt, True)
                lr[j] = val
            sch = StructType(fs)
        return pyref.serialize_example_bytes(sch, tuple(lr))

    frames = []
    for k in range(len(rows)):
        p = {7: {"v_indices": (ArrayType(FloatType()), [1.0])},
             11: {("x_row_splits" if splits else "x_row_lengths"): (ArrayType(FloatType()), [0.0])},
             13: {("x_row_splits" if splits else "x_row_lengths"): (ArrayType(LongType()), [1] if splits else [-1])},
             15: {"e": (ArrayType(FloatType()), [2.0])}}.get(k)
        fr = bytearray(pyref.frame(payload(k, p)))
        if k == 3:
            fr[13] ^= 0x10                                  # a payload byte: TFR_E_CRC_DATA
        if k == 19:
            fr[9] ^= 0x01                                   # the length CRC: a framing error
        frames.append(bytes(fr))
    ds, cidx = CR.with_extras(ws, seed, corrupt)
    shift = lambda i: [j for j, f in enumerate(ds) if f.name == ws[i].name][0]
    return ws, ds, opts, cidx, b"".join(frames), {n: shift(ws.names.index(n)) for n in ("v", "x", "e")}


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_modes_with_every_damage(native, mode, seed):
    flags, pw_mode, resync = MODES[mode]
    ws, ds, opts, cidx, data, at = damaged_case(seed, pw_mode == PW.PERMISSIVE)
    dopts = CR.Opts(opts.vector_format, True, opts.row_splits, True, cidx if pw_mode == PW.PERMISSIVE else None)
    exp = CR.Expect(ds, dopts, data, pw_mode, resync)
    # the restatement sees each damage at its record, reported at the owner
    verd = CR.Expect(ds, dopts, data, PW.PERMISSIVE, True).dropped
    assert [(k, c, f) for k, c, f in verd] == [(3, A.TFR_E_CRC_DATA, -1), (7, A.TFR_E_KIND_MISMATCH, at["v"]),
                                               (11, A.TFR_E_KIND_MISMATCH, at["x"]), (13, A.TFR_E_BAD_NESTING, at["x"]),
                                               (15, A.TFR_E_KIND_MISMATCH, at["e"]), (19, A.TFR_E_CRC_LENGTH, -1)], verd
    dec = decoder(native, ds, dopts, flags)
    try:
        s0 = dec.stats()
        b, _ = dec.decode(np.frombuffer(data, dtype=np.uint8))
        check_batch(b, ds, dopts, exp, f"{mode} seed {seed}")
        if pw_mode == PW.PERMISSIVE:
            h, o = b.unsafe_rows()
            wr, wo = CR.unsafe_rows(ds, exp.rows, dopts)
            assert h.tobytes() == wr.tobytes() and list(o) == list(wo)
        b.release()
        d = delta(s0, dec.stats())
        n_bad = len(exp.dropped) - sum(1 for e in exp.dropped if e[1] in A.FRAMING_ERRORS)
        if pw_mode == PW.DROPMALFORMED:
            assert d["records_dropped"] == n_bad, d
        if pw_mode == PW.PERMISSIVE:
            assert d["records_corrupt"] == n_bad and d["lost_regions"] == (1 if resync else 0), d
        # the tile kernel cannot vouch for the batch, the general path finds the failing records; in the tolerant modes the
        # kept records are decoded again on the tile kernel
        assert d["general_path_batches"] == 1 and d["large_record_batches"] == 0, d
        assert d["count_mode_batches"] == (0 if pw_mode == PW.FAILFAST else 1), d
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# d. views: device columns, host copy, Arrow host and device export, UnsafeRows (sync, async, with partition values)
# ---------------------------------------------------------------------------------------------
_WIDTH = {b"l": 8, b"i": 4, b"f": 4, b"g": 8, b"c": 1, b"s": 2, b"tdD": 4, b"tsu:UTC": 8}


def _arrow_tree(sc, arr, read):
    """an exported Arrow column as nested tuples of its format, length, null count, validity bits and the buffer bytes its
    length covers; read(ptr, nbytes) reads one buffer"""
    fmt, n, off = sc.format, arr.length, arr.offset
    bufs = [arr.buffers[i] for i in range(arr.n_buffers)]

    def bits(ptr):
        return None if not ptr else np.unpackbits(np.frombuffer(read(ptr, (off + n + 7) // 8), np.uint8), bitorder="little")[off:off + n].tolist()

    node = [fmt, n, arr.null_count, bits(bufs[0])]
    if fmt in (b"+l", b"u", b"z"):
        offs = np.frombuffer(read(bufs[1], 4 * (off + n + 1)), np.int32)[off:]
        node.append(offs.tolist())
        if fmt == b"+l":
            child = C.cast(arr.children, C.POINTER(C.POINTER(RI.ArrowArray)))[0].contents
            csc = C.cast(sc.children, C.POINTER(C.POINTER(RI.ArrowSchema)))[0].contents
            node.append(_arrow_tree(csc, child, read))
        else:
            node.append(read(bufs[2], int(offs[-1]))[int(offs[0]):] if n else b"")
    elif fmt == b"b":
        node.append(bits(bufs[1]))
    else:
        w = _WIDTH[fmt]
        node.append(read(bufs[1], w * (off + n))[w * off:])
    return tuple(node)


def arrow_export(native, b, col, device):
    """tfr_batch_export_arrow_host / _device of column col, as _arrow_tree"""
    sc = RI.ArrowSchema()
    if device:
        da = RI.ArrowDeviceArray()
        native._check(native.lib().tfr_batch_export_arrow_device(b.h, col, C.addressof(da), C.addressof(sc)))
        arr = da.array
        assert da.device_type == 2
    else:
        arr = RI.ArrowArray()
        native._check(native.lib().tfr_batch_export_arrow_host(b.h, col, C.addressof(arr), C.addressof(sc)))
    try:
        if device:
            return _arrow_tree(sc, arr, lambda p, nb: BO._dev_array(p, nb, np.uint8).tobytes())
        return _arrow_tree(sc, arr, lambda p, nb: C.string_at(p, nb) if nb else b"")
    finally:
        RI._RELEASE(arr.release)(C.addressof(arr))
        RI._RELEASE(sc.release)(C.addressof(sc))


@pytest.mark.parametrize("seed", [3, 9, 15, 21])
def test_views(native, seed):
    import partition_rows as PR
    from util import assert_columns_equal
    ws, ds, opts = seeded_case(seed, 16)
    rows = CR.seeded_rows(ws, opts, 150, seed)
    data = CR.encode(ws, rows, opts)
    exp = CR.Expect(ds, opts, data, PW.FAILFAST if opts.corrupt is None else PW.PERMISSIVE)
    buf = np.frombuffer(data, dtype=np.uint8)
    want = want_columns(ds, opts, exp.rows)
    dec = decoder(native, ds, opts)
    try:
        s0 = dec.stats()
        b, _ = dec.decode(buf)
        check_batch(b, ds, opts, exp, "host copy")
        host = b.to_host()
        dev = BO.device_columns(b)                         # the device columns, copied from the device as they are
        assert CR.columns_rows(dev, b.n_rows) == want, "device columns"
        assert_columns_equal(dev, host, None, "device columns vs host copy")
        for f, c, h in zip(ds, b.device_columns(), host):  # narrowed columns at their narrow width
            t = I.leaf_id(f.dataType)
            assert c.value_width == h.values.dtype.itemsize, f.name
            if t:
                assert c.elem_type == t and c.value_width == np.dtype(I.TYPES[I.BY_ID[t]][2]).itemsize, f.name
        assert any(I.leaf_id(f.dataType) not in (0, A.TFR_T_TIMESTAMP) for f in ds)
        for col in range(len(host)):                        # the device export holds what the host export holds
            assert arrow_export(native, b, col, True) == arrow_export(native, b, col, False), ("arrow device", col)
        arrs = b.to_arrow()
        assert len(arrs) == len(want[0])
        for i, a in enumerate(arrs):
            assert [CR.canon(v) for v in a.to_pylist()] == [w[i] for w in want], ("arrow", i)
        h, o = b.unsafe_rows()
        wr, wo = CR.unsafe_rows(ds, exp.rows, opts)
        assert h.tobytes() == wr.tobytes() and list(o) == list(wo), "rows"
        rp, op, n, nb = b.unsafe_rows(to_host=False)         # the device rows
        assert n == len(exp.rows) and BO._dev_array(rp, nb, np.uint8).tobytes() == wr.tobytes(), "device rows"
        assert BO._dev_array(op, n + 1, np.int64).tolist() == list(wo), "device row offsets"
        b.release()
        on_path(delta(s0, dec.stats()), "tile", "views")
        ptypes, pvals = ["string", "int", "date"], ["p=1", 7, 19000]
        part = (PR.partition_row(ptypes, pvals), PR.var_flags(ptypes))
        jr, jo = CR.unsafe_rows(ds, exp.rows, opts, ptypes, pvals)
        for asy in (False, True):
            b, _ = dec.decode(buf)
            if asy:
                b.unsafe_rows_async(to_host=True, partition=part)
            h, o = b.unsafe_rows(partition=part)
            assert h.tobytes() == jr.tobytes() and list(o) == list(jo), ("partition", asy)
            b.release()
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# e. count boundaries
# ---------------------------------------------------------------------------------------------
def _encode_all_ways(native, ws, rows, opts, general=False):
    """tfr_encode from columns, tfr_encode_rows and tfr_encode_rows_submit -> their bytes.  `general`: records too large for
    the Example tile emit's shared memory (32 slots of the largest record), which the general emit kernel writes"""
    enc = native.Encoder(ws, 0, **opts.native())
    try:
        out = [enc.encode(A.columns_from_rows(ws, [CR.to_py(ws, r, opts) for r in rows], 0, opts.vector_format))]
        rb, ro = CR.unsafe_rows(ws, rows, opts)
        enc.encode_rows(rb, ro.astype(np.int32))
        out.append(enc.result_host())
        s0 = enc.stats()
        s = enc.submit_rows(rb, ro.astype(np.int32))
        s.wait()
        out.append(s.result_host())
        d = delta(s0, enc.stats())
        assert d["submits"] == 1 and d["general_emit"] == (1 if general else 0), d
        s.release()
        return out
    finally:
        enc.close()


@pytest.mark.parametrize("target", [127, 128, 129])
@pytest.mark.parametrize("big", [False, True], ids=["tile", "large"])
def test_lowered_field_boundary(native, target, big):
    opts = CR.Opts("sparse", True, target % 2 == 0, False)
    ws = CR.boundary_schema(target, opts)
    assert CR.n_lowered(ws, opts) == target
    rows = _with_pad(ws, CR.seeded_rows(ws, opts, 24 if big else 80, target), [12_000] * 8 if big else [])
    data = CR.encode(ws, rows, opts)
    for k, got in enumerate(_encode_all_ways(native, ws, rows, opts, general=big)):
        assert got == data, (target, "encode way", k)
    exp = CR.Expect(ws, opts, data, PW.FAILFAST)
    path = "general" if target > 128 else "large" if big else "tile"
    dec = decoder(native, ws, opts)
    try:
        s0 = dec.stats()
        b, _ = dec.decode(np.frombuffer(data, dtype=np.uint8))
        check_batch(b, ws, opts, exp, f"{target} fields {path}")
        b.release()
        on_path(delta(s0, dec.stats()), path, f"{target} lowered fields")
    finally:
        dec.close()


@pytest.mark.parametrize("n", [64, 65, 128, 129])
def test_narrowed_column_boundary(native, n):
    opts = CR.Opts(ragged=True, extended_types=True)
    ws = CR.narrowed_schema(n)
    assert CR.n_narrowed(ws, opts) == n
    rows = CR.seeded_rows(ws, opts, 70, n)
    data = CR.encode(ws, rows, opts)
    for k, got in enumerate(_encode_all_ways(native, ws, rows, opts)):
        assert got == data, (n, "encode way", k)
    exp = CR.Expect(ws, opts, data, PW.FAILFAST)
    path = "tile" if CR.n_lowered(ws, opts) <= 128 else "general"
    for pipelined in (False, True):
        dec = decoder(native, ws, opts)
        try:
            s0 = dec.stats()
            b, _ = dec.decode(np.frombuffer(data, dtype=np.uint8))
            check_batch(b, ws, opts, exp, f"{n} narrowed")
            b.release()
            on_path(delta(s0, dec.stats()), path, f"{n} narrowed columns")
            if pipelined and path == "tile":
                big = np.frombuffer(CR.encode(ws, rows * 30, opts), dtype=np.uint8)
                bexp = CR.Expect(ws, opts, big.tobytes(), PW.FAILFAST)
                for k in range(3):
                    s0 = dec.stats()
                    b = dec.submit(big)
                    check_batch(b, ws, opts, bexp, f"{n} narrowed, submit {k}")
                    b.release()
                d = delta(s0, dec.stats())
                assert d["speculative_submits"] == 1 and d["speculative_redone"] == 0, d
                assert d["general_path_batches"] == 0 and d["large_record_batches"] == 0, d
        finally:
            dec.close()


# ---------------------------------------------------------------------------------------------
# f. encode: three ways, a pipelined stream with an outlier, the malformed-input rules
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 6, 13, 19])
def test_encode_three_ways_and_back(native, seed):
    ws, _, opts = seeded_case(seed, 20)
    opts = CR.Opts(opts.vector_format, True, opts.row_splits, True)       # (the writer's schema has no corrupt-record column)
    rows = _with_pad(ws, CR.seeded_rows(ws, opts, 400, seed), [])
    data = CR.encode(ws, rows, opts)
    for k, got in enumerate(_encode_all_ways(native, ws, rows, opts)):
        assert got == data, (seed, "encode way", k)
    dec = decoder(native, ws, opts)
    try:
        b, _ = dec.decode(np.frombuffer(data, dtype=np.uint8))
        back = [[c.get(r) for c in b.to_host()] for r in range(b.n_rows)]
        assert [CR.canon(x) for x in back] == [CR.canon(list(CR.column_row(ws, r, opts))) for r in rows]
        b.release()
    finally:
        dec.close()


@pytest.mark.parametrize("seed", [5, 6])
def test_encode_submit_steady_and_outlier(native, seed):
    ws, ds, opts = seeded_case(seed, 16)
    flushes = []
    for k in range(5):
        rows = CR.seeded_rows(ws, opts, 3000, seed * 10 + k)
        rows = _with_pad(ws, rows, [2] * 1500 + [3_000] if k == 3 else [])      # flush 3: one record 30x the others
        rb, ro = CR.unsafe_rows(ws, rows, opts)
        flushes.append((rb, ro.astype(np.int32), CR.encode(ws, rows, opts)))
    enc = native.Encoder(ws, 0, **opts.native())
    try:
        stats = []
        for rb, ro, want in flushes:
            s = enc.submit_rows(rb, ro)
            s.wait()
            assert s.result_host() == want
            s.release()
            stats.append(enc.stats())
        d_out = delta(stats[2], stats[3])
        d_after = delta(stats[3], stats[4])
        assert stats[2]["speculative_submits"] >= 1 and stats[2]["speculative_redone"] == 0, stats[2]
        assert d_out["speculative_submits"] == 1 and d_out["speculative_redone"] == 1, d_out
        assert d_after["speculative_submits"] == 1 and d_after["speculative_redone"] == 0, d_after
    finally:
        enc.close()


def _write_error(native, ws, rows, opts, via, patch=None):
    enc = native.Encoder(ws, 0, **opts.native())
    try:
        if via == "columns":
            cols = A.columns_from_rows(ws, [CR.to_py(ws, r, opts) for r in rows], 0, opts.vector_format)
            if patch:
                patch(cols)
            enc.encode(cols)
        else:
            rb, ro = CR.unsafe_rows(ws, rows, opts)
            enc.encode_rows(rb, ro.astype(np.int32))
    except native.TfrError as e:
        return type(e).__name__, e.code, e.row, e.field   # (the encoders report a row only: field is -1)
    finally:
        enc.close()
    return None


@pytest.mark.parametrize("rule", ["sparse_struct", "ragged_offsets", "null_inner_array"])
def test_malformed_input_fails_as_with_the_feature_alone(native, rule):
    opts = CR.Opts("sparse", True, False, True)
    ws = CR.seeded_schema(8, 16, opts)
    fields = list(ws.fields)
    fields.insert(5, CR.make_field("v", "vector", True))
    fields.insert(9, CR.make_field("x", "long:2", True))
    ws = StructType(fields)
    rows = [list(r) for r in CR.seeded_rows(ws, opts, 12, 8)]
    for r in rows:
        r[9] = [[1, 2], [3]]
        r[5] = DenseVector([1.0])
    bad = 6
    via, patch = "rows", None
    if rule == "sparse_struct":
        rows[bad][5] = V.RawVector(V.struct_bytes(0, -1, V.int_array([]), V.double_array([])))
    elif rule == "null_inner_array":
        rows[bad][9] = [[1], None, [2]]
    else:
        via = "columns"
    rows = [tuple(r) for r in rows]
    idx = 5 if rule == "sparse_struct" else 9
    alone = StructType([ws[idx]])

    def patch_at(col_index):
        def p(cols):
            c = cols[col_index]
            c.offsets[1][int(c.offsets[0][bad])] = 50    # row bad - 1's last list runs on, row bad's first is negative
        return p

    got = _write_error(native, ws, rows, opts, via, patch_at(idx) if via == "columns" else None)
    want = _write_error(native, alone, [(r[idx],) for r in rows], opts, via, patch_at(0) if via == "columns" else None)
    assert want is not None and got == want, (rule, got, want)
