"""GPU tests of extendedTypes=true (include/tfrgpu.h, INT64 TYPES), through tests/int64_types.py.  A write -- tfr_encode,
tfr_encode_rows and tfr_encode_rows_submit -- is pyref's encoding of the LongType rows with the widened values.  A read is the
LongType decode of the same bytes, narrowed in numpy: the oracle's (oracle/tfr_oracle.c) for Example and SequenceExample records
in FAILFAST and, with the failing frames cut out, DROPMALFORMED; this library's own LongType decode (itself tested against the
oracle elsewhere) for ragged fields, PERMISSIVE and resync, which the oracle does not read.  Paths: tile, large-record, general
(asserted through the decoder's counters) and the pipelined submit."""
import ctypes as C
import datetime as dt
import os

import numpy as np
import pytest

import int64_types as I
import test_gpu_batch_outputs as BO
from test_gpu_row_index import ArrowDeviceArray, ArrowSchema, ArrowArray, _RELEASE
from oracle import oracle, pyref
from spark_tfrecord_b200 import _cabi as A
from spark_tfrecord_b200.sqltypes import *  # noqa

pytestmark = pytest.mark.gpu
NAMES = list(I.TYPES)


@pytest.fixture(scope="module")
def native():
    from spark_tfrecord_b200 import _native
    _native.lib()
    return _native


def _gen(rng, name):
    """a narrow leaf value of type `name` (an int, as its column holds it)"""
    t = I.TYPES[name][1]
    if t == A.TFR_T_BOOL:
        return int(rng.integers(0, 2))
    # dates and timestamps inside what datetime.date / datetime.datetime hold (years 1 to 9999)
    lo, hi = {A.TFR_T_INT8: (-128, 128), A.TFR_T_INT16: (-32768, 32768), A.TFR_T_DATE: (-719162, 2932897)}.get(
        t, (-62135596800 * 10**6, 253402300799 * 10**6))
    return int(rng.integers(lo, hi))


def _schema(name, nullable, depth):
    et = I.TYPES[name][0]
    for _ in range(depth):
        et = ArrayType(et)
    return StructType([StructField("id", LongType(), False), StructField("x", et, nullable), StructField("w", FloatType(), True)])


def _rows(name, nullable, depth, n=257, seed=0):
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        if nullable and i % 5 == 0:
            x = None
        elif depth == 0:
            x = _gen(rng, name)
        elif depth == 1:
            x = [_gen(rng, name) for _ in range(int(rng.integers(0, 13)))]
        else:
            x = [[_gen(rng, name) for _ in range(int(rng.integers(0, 5)))] for _ in range(int(rng.integers(0, 6)))]
        rows.append((i, x, float(i)))
    return rows


def _pyref_bytes(schema, rows, rt=0, ragged=False):
    low = I.long_schema(schema)
    lr = I.long_rows(schema, rows)
    if ragged:
        import ragged_rows as RR
        return RR.encode(low, lr)
    ser = pyref.serialize_sequence_example_bytes if rt == 1 else pyref.serialize_example_bytes
    return b"".join(pyref.frame(ser(low, r)) for r in lr)


def _py(schema, row):
    """a row of narrow ints as the Python values the writer takes (bool, int, date, aware datetime)"""
    out = []
    for f, v in zip(schema, row):
        t = I.leaf_id(f.dataType)
        conv = (lambda x: A.int64_value(t, x)) if t else (lambda x: x)
        out.append(None if v is None else [conv(e) if not isinstance(e, list) else [conv(y) for y in e] for e in v] if isinstance(v, list) else conv(v))
    return out


# ---------------------------------------------------------------------------------------------
# write: tfr_encode's bytes are pyref's of the LongType rows
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("layout", ["d0", "d1", "seq", "ragged"])
def test_encode_bytes_equal_pyref(native, name, nullable, layout):
    depth = {"d0": 0, "d1": 1, "seq": 2, "ragged": 2}[layout]
    rt = 1 if layout == "seq" else 0
    sch = _schema(name, nullable, depth)
    rows = _rows(name, nullable, depth, seed=depth)
    enc = native.Encoder(sch, rt, extended_types=True, ragged=layout == "ragged")
    try:
        got = enc.encode(A.columns_from_rows(sch, [tuple(_py(sch, r)) for r in rows], rt))
    finally:
        enc.close()
    assert got == _pyref_bytes(sch, rows, rt, layout == "ragged")


def test_encode_bool_byte_nonzero_writes_one(native):
    sch = StructType([StructField("b", BooleanType(), False), StructField("a", ArrayType(BooleanType()), False)])
    n = 6
    raw = np.array([0, 1, 2, 0xFF, 0x80, 0], dtype=np.uint8)
    c0 = A.HostColumn(A.TFR_T_BOOL, 0, n, None, [], raw)
    c1 = A.HostColumn(A.TFR_T_BOOL, 1, n, None, [np.arange(n + 1, dtype=np.int32)], raw)
    enc = native.Encoder(sch, 0, extended_types=True)
    try:
        got = enc.encode([c0, c1])
    finally:
        enc.close()
    want = [(1 if v else 0, [1 if v else 0]) for v in raw.tolist()]
    assert got == b"".join(pyref.frame(pyref.serialize_example_bytes(I.long_schema(sch), r)) for r in want)


def test_encode_needs_value_width(native):
    sch = StructType([StructField("s", ShortType(), False)])
    c = A.HostColumn(A.TFR_T_INT64, 0, 3, None, [], np.array([1, 2, 3], np.int64)).to_ctypes()   # an int64 column: width 8
    enc = native.Encoder(sch, 0, extended_types=True)
    try:
        with pytest.raises(native.TfrError) as e:
            enc.encode_columns([c], False)
        assert e.value.code == A.TFR_E_INVALID_ARG
    finally:
        enc.close()


def _row_batch(sch, rows):
    rb = [I.unsafe_row(sch, r) for r in rows]
    offs = np.concatenate([[0], np.cumsum([len(x) for x in rb])]).astype(np.int32)
    return np.frombuffer(b"".join(rb), dtype=np.uint8).copy(), offs


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("layout", ["d0", "d1", "seq", "ragged"])
def test_encode_rows_bytes_equal_pyref(native, name, nullable, layout):
    """tfr_encode_rows and tfr_encode_rows_submit read the narrow UnsafeRow slots and elements (a boolean byte != 0)"""
    depth = {"d0": 0, "d1": 1, "seq": 2, "ragged": 2}[layout]
    rt = 1 if layout == "seq" else 0
    sch = _schema(name, nullable, depth)
    rows = _rows(name, nullable, depth, seed=depth + 10)
    if I.TYPES[name][1] == A.TFR_T_BOOL:                  # boolean bytes of 2 and 0xFF in the rows write 1
        mark = lambda v, k: None if v is None else [mark(e, k) for e in v] if isinstance(v, list) else (k if v else 0)
        rows = [(i, mark(x, 2 if i % 2 else 0xFF) if i % 3 else x, w) for i, x, w in rows]
    want = _pyref_bytes(sch, rows, rt, layout == "ragged")
    buf, offs = _row_batch(sch, rows)
    enc = native.Encoder(sch, rt, extended_types=True, ragged=layout == "ragged")
    try:
        enc.encode_rows(buf, offs, on_device=False)
        assert enc.result_host() == want
        for _ in range(4):                                  # pipelined: the encoder learns, then submits without a host wait
            h = enc.submit_rows(buf, offs, on_device=False)
            h.wait()
            assert h.result_host() == want
            h.release()
    finally:
        enc.close()


# ---------------------------------------------------------------------------------------------
# read: the oracle's LongType decode, narrowed
# ---------------------------------------------------------------------------------------------
def _edge_rows(depth, n=203, seed=1):
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        if i % 9 == 4:
            x = None
        elif depth == 0:
            x = I.EDGES[i % len(I.EDGES)]
        elif depth == 1:
            x = [I.EDGES[int(k)] for k in rng.integers(0, len(I.EDGES), int(rng.integers(0, 11)))]
        else:
            x = [[I.EDGES[int(k)] for k in rng.integers(0, len(I.EDGES), int(rng.integers(0, 4)))] for _ in range(int(rng.integers(0, 5)))]
        rows.append((i, x, float(i)))
    return rows


def _long_bytes(long_sch, rows, rt=0):
    ser = pyref.serialize_sequence_example_bytes if rt == 1 else pyref.serialize_example_bytes
    return b"".join(pyref.frame(ser(long_sch, r)) for r in rows)


def _check_batch(b, sch, want_cols, info=None):
    if info is not None:
        for k in ("n_rows", "error_code", "error_row", "error_field"):
            assert b.info[k] == info[k], (k, b.info, info)
    got = b.to_host()
    dev = b.device_columns()
    for i, (f, g, w) in enumerate(zip(sch, got, want_cols)):
        t = I.leaf_id(f.dataType)
        want_vals = I.narrow(t, w.values) if t else w.values
        assert g.elem_type == (t or w.elem_type), (f.name, g.elem_type)
        assert dev[i].elem_type == g.elem_type
        if t:
            assert dev[i].value_width == np.dtype(I.TYPES[I.BY_ID[t]][2]).itemsize
        assert g.n_rows == w.n_rows
        np.testing.assert_array_equal(np.unpackbits(g.validity, bitorder="little")[:g.n_rows],
                                      np.unpackbits(w.validity, bitorder="little")[:w.n_rows], err_msg=f.name)
        assert len(g.offsets) == len(w.offsets)
        for go, wo in zip(g.offsets, w.offsets):
            np.testing.assert_array_equal(go, wo, err_msg=f.name)
        np.testing.assert_array_equal(g.values, want_vals.astype(g.values.dtype), err_msg=f.name)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("layout", ["d0", "d1", "seq", "ragged"])
def test_decode_edges_tile_and_pipelined(native, name, layout):
    depth = {"d0": 0, "d1": 1, "seq": 2, "ragged": 2}[layout]
    rt = 1 if layout == "seq" else 0
    sch = _schema(name, True, depth)
    low = I.long_schema(sch)
    rows = _edge_rows(depth)
    if layout == "ragged":
        import ragged_rows as RR
        data = RR.encode(low, rows)
        want = [native.Decoder(low, 0, ragged=True)]
        try:
            b = want[0].decode(data)[0]
            want_cols = b.to_host()
            b.release()
        finally:
            want[0].close()
    else:
        data = _long_bytes(low, rows, rt)
        want_cols = oracle.decode(data, low, rt).columns
    dec = native.Decoder(sch, rt, extended_types=True, ragged=layout == "ragged")
    try:
        b, used = dec.decode(data)
        assert used == len(data)
        _check_batch(b, sch, want_cols)
        b.release()
        big = data * 40                                          # pipelined: shapes learned, then submits with no host sync
        if layout == "ragged":                                   # (narrow_kernel behind ragged_assemble_kernel on the submit stream)
            ref = native.Decoder(low, 0, ragged=True)
            try:
                w = ref.decode(big)[0]
                want_big = w.to_host()
                w.release()
            finally:
                ref.close()
        else:
            want_big = oracle.decode(big, low, rt).columns
        for _ in range(3):
            b = dec.submit(big)
            _check_batch(b, sch, want_big)
            b.release()
        assert dec.stats()["speculative_submits"] >= 1
    finally:
        dec.close()


@pytest.mark.parametrize("name", NAMES)
def test_decode_large_records(native, name):
    sch = StructType([StructField("x", ArrayType(I.TYPES[name][0]), True), StructField("pad", BinaryType(), True),
                      StructField("s", I.TYPES[name][0], True)])
    low = I.long_schema(sch)
    rng = np.random.default_rng(5)
    rows = [([I.EDGES[int(k)] for k in rng.integers(0, len(I.EDGES), 50)], bytes(100_000 + i), I.EDGES[i % len(I.EDGES)])
            for i in range(40)]
    data = _long_bytes(low, rows)
    want = oracle.decode(data, low).columns
    dec = native.Decoder(sch, 0, extended_types=True)
    try:
        for it in range(4):
            b = dec.submit(data) if it else dec.decode(data)[0]
            _check_batch(b, sch, want)
            b.release()
        assert dec.stats()["large_record_batches"] >= 1, dec.stats()
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# the modes: a FloatList in a BooleanType field is a kind mismatch at that field
# ---------------------------------------------------------------------------------------------
def _mode_data(low, rows, bad_at, resync_at=None):
    parts = []
    for i, r in enumerate(rows):
        if i in bad_at:
            parts.append(pyref.frame(pyref.example({"id": pyref.int64_feature(i), "x": pyref.float_feature(1.5)}).SerializeToString()))
        else:
            parts.append(pyref.frame(pyref.serialize_example_bytes(low, r)))
        if resync_at is not None and i == resync_at:
            parts.append(b"\x07" * 23)                           # a framing error, then the next verified frame
    return b"".join(parts)


@pytest.mark.parametrize("mode", ["FAILFAST", "DROPMALFORMED", "PERMISSIVE", "DROPMALFORMED+resync", "PERMISSIVE+resync"])
def test_modes_kind_mismatch(native, mode):
    sch = StructType([StructField("id", LongType(), False), StructField("x", BooleanType(), True),
                      StructField("d", ArrayType(DateType()), True)])
    low = I.long_schema(sch)
    rows = [(i, I.EDGES[i % len(I.EDGES)], [I.EDGES[(i + k) % len(I.EDGES)] for k in range(i % 4)]) for i in range(300)]
    resync = mode.endswith("+resync")
    data = _mode_data(low, rows, {7, 150, 151}, 200 if resync else None)
    flags = A.TFR_F_DEFAULT | {"FAILFAST": 0, "DROPMALFORMED": A.TFR_F_DROP_MALFORMED, "PERMISSIVE": A.TFR_F_PERMISSIVE}[mode.split("+")[0]]
    if resync:
        flags |= A.TFR_F_RESYNC
    # the expectation: the LongType decode of the same bytes in the same mode (the oracle reads FAILFAST only)
    ref = native.Decoder(low, 0, 0, flags)
    dec = native.Decoder(sch, 0, 0, flags, extended_types=True)
    try:
        w, _ = ref.decode(data)
        want_cols, want_info, want_dropped = w.to_host(), dict(w.info), w.dropped()
        w.release()
        if mode == "FAILFAST":
            assert want_info["error_code"] == A.TFR_E_KIND_MISMATCH and want_info["error_row"] == 7 and want_info["error_field"] == 1
            np.testing.assert_array_equal(oracle.decode(data, low).columns[1].values, want_cols[1].values)
        else:
            assert [d[0] for d in want_dropped if d[2] == A.TFR_E_KIND_MISMATCH] == [7, 150, 151] or resync
        if mode == "DROPMALFORMED":                                # the oracle on the records that do not fail
            clean = _mode_data(low, [r for i, r in enumerate(rows) if i not in (7, 150, 151)], set())
            for w, o in zip(want_cols, oracle.decode(clean, low).columns):
                np.testing.assert_array_equal(w.values, o.values)
                for wo, oo in zip(w.offsets, o.offsets):
                    np.testing.assert_array_equal(wo, oo)
        g0 = dec.stats()["general_path_batches"]
        b, _ = dec.decode(data)
        _check_batch(b, sch, want_cols, want_info)
        assert b.dropped() == want_dropped
        assert dec.stats()["general_path_batches"] > g0          # the failing records send the batch to the general path
        b.release()
    finally:
        ref.close(); dec.close()


# ---------------------------------------------------------------------------------------------
# views: Arrow formats, the boolean bitmap, UnsafeRows
# ---------------------------------------------------------------------------------------------
def _arrow(native, b, col, device):
    sc = ArrowSchema()
    if device:
        da = ArrowDeviceArray()
        native._check(native.lib().tfr_batch_export_arrow_device(b.h, col, C.addressof(da), C.addressof(sc)))
        arr, rel = da.array, da
    else:
        arr = ArrowArray()
        native._check(native.lib().tfr_batch_export_arrow_host(b.h, col, C.addressof(arr), C.addressof(sc)))
        rel = arr
    return sc, arr, rel


@pytest.mark.parametrize("n", [1, 7, 9, 100, 1001])
@pytest.mark.parametrize("device", [False, True])
def test_arrow_formats_and_bitmap(native, n, device):
    sch = StructType([StructField(nm, t[0], True) for nm, t in I.TYPES.items()] +
                     [StructField("ab", ArrayType(BooleanType()), True)])
    low = I.long_schema(sch)
    rng = np.random.default_rng(n)
    rows = [tuple(None if (i + j) % 6 == 5 else int(I.EDGES[int(rng.integers(0, len(I.EDGES)))]) for j in range(5)) +
            ([I.EDGES[int(k)] for k in rng.integers(0, len(I.EDGES), int(rng.integers(0, 12)))],) for i in range(n)]
    data = _long_bytes(low, rows)
    want = oracle.decode(data, low).columns
    dec = native.Decoder(sch, 0, extended_types=True)
    try:
        b, _ = dec.decode(data)
        for col, (nm, t) in enumerate(list(I.TYPES.items()) + [("ab", I.TYPES["bool"])]):
            sc, arr, rel = _arrow(native, b, col, device)
            try:
                if nm == "ab":
                    assert sc.format == b"+l"
                    child = C.cast(arr.children, C.POINTER(C.POINTER(ArrowArray)))[0].contents
                    m = int(child.length)
                    assert m == len(want[col].values)
                    buf = child.buffers[1]
                else:
                    assert sc.format.decode() == t[3]
                    m = n
                    buf = arr.buffers[1]
                vals = I.narrow(t[1], want[col].values)
                if t[1] == A.TFR_T_BOOL:
                    nb = (m + 7) // 8
                    got = BO._dev_array(buf, nb, np.uint8) if device else np.ctypeslib.as_array(C.cast(buf, C.POINTER(C.c_uint8)), (nb,)).copy() if nb else np.zeros(0, np.uint8)
                    np.testing.assert_array_equal(got, np.packbits(vals, bitorder="little"), err_msg=f"{nm} n={n}")
                else:
                    got = BO._dev_array(buf, m, vals.dtype) if device else np.ctypeslib.as_array(C.cast(buf, C.POINTER(C.c_uint8)), (m * vals.itemsize,)).view(vals.dtype).copy()
                    np.testing.assert_array_equal(got, vals, err_msg=nm)
            finally:
                _RELEASE(arr.release)(C.addressof(arr))
                _RELEASE(sc.release)(C.addressof(sc))
        b.release()
    finally:
        dec.close()


def _row_schema():
    return StructType([StructField("id", LongType(), False)] + [StructField(nm, t[0], True) for nm, t in I.TYPES.items()] +
                      [StructField("a_" + nm, ArrayType(t[0]), True) for nm, t in I.TYPES.items()])


@pytest.mark.parametrize("variant", ["sync", "partition", "async"])
def test_unsafe_rows_layout(native, variant):
    sch = _row_schema()
    low = I.long_schema(sch)
    rng = np.random.default_rng(3)
    rows = []
    for i in range(300):
        sc = [None if (i + j) % 7 == 3 else I.EDGES[int(rng.integers(0, len(I.EDGES)))] for j in range(5)]
        ar = [None if (i + j) % 8 == 1 else [I.EDGES[int(k)] for k in rng.integers(0, len(I.EDGES), int(rng.integers(0, 20)))] for j in range(5)]
        rows.append(tuple([i] + sc + ar))
    data = _long_bytes(low, rows)
    want_cols = oracle.decode(data, low).columns
    nar = []
    for r in range(len(rows)):
        nar.append(tuple(c.get(r) for c in want_cols))
    ids = [I.leaf_id(f.dataType) for f in sch]
    def nrow(row):
        out = []
        for t, v in zip(ids, row):
            if t and v is not None:
                v = [int(I.narrow(t, [e])[0]) for e in v] if isinstance(v, list) else int(I.narrow(t, [v])[0])
            out.append(v)
        return out
    want_rows = [I.unsafe_row(sch, nrow(r)) for r in nar]
    part = None
    if variant == "partition":
        part_row = np.zeros(24, np.uint8); part_row[8] = 1; part_row[16] = 0x7F    # BooleanType, ByteType partition values
        part = (part_row.tobytes(), [0, 0])
    dec = native.Decoder(sch, 0, extended_types=True)
    try:
        for it in range(3 if variant == "async" else 1):
            b = dec.submit(data * 4) if variant == "async" else dec.decode(data)[0]
            if variant == "async":
                b.unsafe_rows_async(True)
            buf, offs = b.unsafe_rows(True, part)
            reps = 4 if variant == "async" else 1
            assert len(offs) == len(rows) * reps + 1
            for r in range(len(rows) * reps):
                got = buf[offs[r]:offs[r + 1]].tobytes()
                w = want_rows[r % len(rows)]
                if part is not None:
                    nf, np_ = len(sch.fields), 2
                    nw = (nf + np_ + 63) // 64
                    wb = bytearray(8 * nw + 8 * (nf + np_))
                    wb[0:8] = w[0:8]
                    wb[8 * nw: 8 * nw + 8 * nf] = w[8:8 + 8 * nf]
                    wb[8 * nw + 8 * nf:] = part[0][8:24]
                    var = bytearray(w[8 + 8 * nf:])
                    # the data fields' variable region moves by the two partition slots: relocate the array slots
                    for j, f in enumerate(sch):
                        s = int.from_bytes(wb[8 * nw + 8 * j: 8 * nw + 8 * j + 8], "little")
                        if isinstance(f.dataType, ArrayType) and s:
                            s += 16 << 32
                            wb[8 * nw + 8 * j: 8 * nw + 8 * j + 8] = s.to_bytes(8, "little")
                    w = bytes(wb) + bytes(var)
                assert got == w, (variant, r)
            b.release()
    finally:
        dec.close()


# ---------------------------------------------------------------------------------------------
# end to end: DefaultSource with the option; inferSchema gives LongType
# ---------------------------------------------------------------------------------------------
def test_default_source_round_trip(native, tmp_path):
    from spark_tfrecord_b200 import io
    utc = dt.timezone.utc
    sch = StructType([StructField("b", BooleanType(), True), StructField("y", ByteType(), True), StructField("s", ShortType(), True),
                      StructField("d", DateType(), True), StructField("t", TimestampType(), True),
                      StructField("ad", ArrayType(DateType()), True), StructField("ab", ArrayType(BooleanType()), True)])
    rows = [(True, -128, 32767, dt.date(1969, 12, 31), dt.datetime(2024, 2, 29, 12, 0, 0, 123456, tzinfo=utc),
             [dt.date(2000, 1, 1), dt.date(1970, 1, 1)], [True, False, True]),
            (None, None, None, None, None, None, None),
            (False, 5, -3, dt.date(2038, 1, 19), dt.datetime(1900, 1, 1, tzinfo=utc), [], [])]
    opts = {"extendedTypes": "true"}
    path = str(tmp_path / "part-0.tfrecord")
    w = io.DefaultSource().prepareWrite(opts, sch).newInstance(path, sch)
    for r in rows:
        w.write(r)
    w.close()
    got = list(io.DefaultSource().buildReader(sch, sch, opts)(io.PartitionedFile(path)))
    assert [tuple(r) for r in got] == rows
    inferred = io.DefaultSource().inferSchema(opts, [path])
    assert {f.name: f.dataType for f in inferred} == {**{k: LongType() for k in "bysdt"}, "ad": ArrayType(LongType()),
                                                     "ab": ArrayType(LongType())}
    # a naive datetime is refused
    w = io.DefaultSource().prepareWrite(opts, sch).newInstance(str(tmp_path / "part-1.tfrecord"), sch)
    with pytest.raises(ValueError):
        w.write((None, None, None, None, dt.datetime(2020, 1, 1), None, None))
        w.close()
