"""nestedArrayFormat=ragged on one GPU.  A seeded corpus of Example records (id: long, x: ragged long with 4-32 inner lists of
0-8 ids, y: ragged float with 4-32 inner lists of 0-8 values, w: float, k: int), built as numpy columns, is encoded once by the
ragged encoder.  Before any time is reported every output is checked:
  - the first 2,000 records are byte-identical to oracle/pyref's encoding of the lowered rows (tests/ragged_rows.py);
  - the ragged decode gives back the input columns, and the plain decode (the same bytes read as x_values, x_row_lengths, ...)
    gives the lowered columns;
  - tfr_encode_rows of the decoded batch's UnsafeRows gives the same bytes as tfr_encode of the columns.
Then, the arms alternated rep by rep after a warm-up (medians, CUDA events around each synchronous call):
  - resident decode GB/s (device input) with the ragged schema, and with the two plain fields per ragged field;
  - the assembly kernel's time (torch.profiler, a run of its own);
  - encode GB/s of framed output for host columns (tfr_encode) and for host UnsafeRows (tfr_encode_rows).
Prints one JSON line with the card's name and power limit, read in the same call.

--partition rowSplits (raggedPartition=rowSplits) checks the same outputs for the row-splits layout too (bytes against
tests/ragged_splits_rows.py, the ragged decode, the plain decode's splits part, tfr_encode_rows), then alternates the lengths
and the splits layout on the same records: resident decode, the assembly kernels' time (ragged_*), and tfr_encode of columns."""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--partition", choices=["rowLengths", "rowSplits"], default="rowLengths")
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(HERE, ".."))
    sys.path.insert(0, os.path.join(HERE, "..", "tests"))
    import numpy as np
    import torch
    import ragged_rows as RR
    from spark_tfrecord_b200 import _native
    from spark_tfrecord_b200._cabi import HostColumn, TFR_T_FLOAT32, TFR_T_FLOAT64, TFR_T_INT32, TFR_T_INT64
    from spark_tfrecord_b200.sqltypes import (ArrayType, FloatType, IntegerType, LongType, StructField, StructType)

    n = a.records
    rng = np.random.default_rng(0)
    sch = StructType([StructField("id", LongType(), False), StructField("x", ArrayType(ArrayType(LongType())), True),
                      StructField("y", ArrayType(ArrayType(FloatType())), True), StructField("w", FloatType(), True),
                      StructField("k", IntegerType(), True)])

    def ragged(kind):
        inner = rng.integers(4, 33, n)
        off0 = np.concatenate([[0], np.cumsum(inner)]).astype(np.int32)
        lens = rng.integers(0, 9, int(off0[-1]))
        off1 = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        vals = (rng.integers(0, 1 << 30, int(off1[-1])) if kind == TFR_T_INT64 else
                rng.standard_normal(int(off1[-1])).astype(np.float32))
        return HostColumn(kind, 2, n, None, [off0, off1.astype(np.int32)], vals)

    cols = [HostColumn(TFR_T_INT64, 0, n, None, [], np.arange(n, dtype=np.int64)), ragged(TFR_T_INT64), ragged(TFR_T_FLOAT32),
            HostColumn(TFR_T_FLOAT32, 0, n, None, [], rng.standard_normal(n).astype(np.float32)),
            HostColumn(TFR_T_INT32, 0, n, None, [], rng.integers(-1000, 1000, n).astype(np.int32))]
    enc = _native.Encoder(sch, 0, ragged=True)
    data = enc.encode(cols)
    # ---- checks ----
    m = min(n, 2000)
    first = [tuple(c.get(r) for c in cols) for r in range(m)]
    first = [(r[0], r[1], [[float(np.float32(v)) for v in i] for i in r[2]], r[3], r[4]) for r in first]
    ref = RR.encode(sch, first)
    assert data[:len(ref)] == ref, "encoded bytes differ from the restatement"
    dev = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    dec_r = _native.Decoder(sch, 0, ragged=True)
    dec_p = _native.Decoder(RR.lowered_schema(sch), 0)
    b, _ = dec_r.decode(dev)
    got = b.to_host()
    assert b.info["error_code"] == 0 and b.n_rows == n
    for c, g in zip(cols, got):
        assert all(np.array_equal(o, go) for o, go in zip(c.offsets, g.offsets)) and np.array_equal(c.values, g.values)
    rows, offs = b.unsafe_rows()
    rows, offs = rows.copy(), offs.astype(np.int32)
    b.release()
    b, _ = dec_p.decode(dev)
    got = b.to_host()
    for j, c in ((1, cols[1]), (2, cols[2])):
        assert np.array_equal(got[j].offsets[0], c.offsets[1][c.offsets[0]]) and np.array_equal(got[j].values, c.values)
        ln = got[4 + j]
        assert np.array_equal(ln.offsets[0], c.offsets[0]) and np.array_equal(ln.values, np.diff(c.offsets[1]))
    b.release()
    enc.encode_rows(rows, offs)
    assert enc.result_host() == data, "UnsafeRows encode differs from the columns encode"

    if a.partition == "rowSplits":
        return splits_arm(a, sch, cols, data, dev, dec_r, enc)

    # ---- times ----
    def timed(f):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        f()
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / 1e3

    def dec_once(d):
        bb, _ = d.decode(dev)
        bb.wait()
        bb.release()

    arms = {"decode_ragged": lambda: dec_once(dec_r), "decode_plain": lambda: dec_once(dec_p),
            "encode_columns": lambda: enc.encode(cols), "encode_rows": lambda: enc.encode_rows(rows, offs)}
    for f in arms.values():
        f(); f()
    t = {k: [] for k in arms}
    for _ in range(a.reps):
        for k, f in arms.items():
            t[k].append(timed(f))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dec_once(dec_r)
    asm = sum(ev.device_time_total for ev in prof.key_averages() if "ragged_assemble_kernel" in ev.key) / 1e3
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    med = {k: statistics.median(v) for k, v in t.items()}
    print(json.dumps({"gpu": gpu, "records": n, "framed_bytes": len(data), "checked": True,
                      "decode_ragged_GBps": len(data) / med["decode_ragged"] / 1e9,
                      "decode_plain_GBps": len(data) / med["decode_plain"] / 1e9,
                      "assembly_ms": asm, "decode_ragged_ms": med["decode_ragged"] * 1e3,
                      "encode_columns_GBps": len(data) / med["encode_columns"] / 1e9,
                      "encode_rows_GBps": len(data) / med["encode_rows"] / 1e9}))


def _timed(torch, f):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    f()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / 1e3


def splits_arm(a, sch, cols, data_len, dev_len, dec_len, enc_len):
    """--partition rowSplits: the row-splits layout checked, then timed against the lengths layout on the same records"""
    import numpy as np
    import torch
    import ragged_splits_rows as RS
    from spark_tfrecord_b200 import _cabi as A
    from spark_tfrecord_b200 import _native
    n = a.records
    enc = _native.Encoder(sch, 0, ragged=True, row_splits=True)
    data = enc.encode(cols)
    m = min(n, 2000)
    first = [tuple(c.get(r) for c in cols) for r in range(m)]
    first = [(r[0], r[1], [[float(np.float32(v)) for v in i] for i in r[2]], r[3], r[4]) for r in first]
    ref = RS.encode(sch, first)
    assert data[:len(ref)] == ref, "row-splits bytes differ from the restatement"
    dev = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    dec = _native.Decoder(sch, 0, ragged=True, row_splits=True)
    b, _ = dec.decode(dev)
    got = b.to_host()
    assert b.info["error_code"] == 0 and b.n_rows == n
    for c, g in zip(cols, got):
        assert all(np.array_equal(o, go) for o, go in zip(c.offsets, g.offsets)) and np.array_equal(c.values, g.values)
    rows, offs = b.unsafe_rows()
    rows, offs = rows.copy(), offs.astype(np.int32)
    b.release()
    dec_p = _native.Decoder(RS.lowered_schema(sch), 0)
    b, _ = dec_p.decode(dev)
    got = b.to_host()
    for j, c in ((1, cols[1]), (2, cols[2])):
        sp = got[4 + j]
        assert np.array_equal(sp.offsets[0], c.offsets[0] + np.arange(n + 1)), "one more entry per row"
        o0, o1 = c.offsets[0].astype(np.int64), c.offsets[1].astype(np.int64)
        k = np.diff(o0) + 1                                            # entries per row
        row = np.repeat(np.arange(n), k)
        at = np.arange(int(k.sum())) - np.repeat(np.cumsum(k) - k, k) + o0[row]
        want = o1[at] - o1[o0[row]]
        assert np.array_equal(sp.values, want)
    b.release()
    dec_p.close()
    enc.encode_rows(rows, offs)
    assert enc.result_host() == data, "UnsafeRows encode differs from the columns encode"
    # the other partition's file: every record fails at x
    b, _ = dec.decode(dev_len)
    assert (b.info["error_code"], b.info["error_row"], b.info["error_field"]) == (A.TFR_E_BAD_NESTING, 0, 1)
    b.release()

    def dec_once(d, x):
        bb, _ = d.decode(x)
        bb.wait()
        bb.release()

    arms = {"decode_lengths": lambda: dec_once(dec_len, dev_len), "decode_splits": lambda: dec_once(dec, dev),
            "encode_lengths": lambda: enc_len.encode(cols), "encode_splits": lambda: enc.encode(cols)}
    for f in arms.values():
        f(); f()
    t = {k: [] for k in arms}
    for _ in range(a.reps):
        for k, f in arms.items():
            t[k].append(_timed(torch, f))
    from torch.profiler import ProfilerActivity, profile
    asm = {}
    for k, d, x in (("lengths", dec_len, dev_len), ("splits", dec, dev)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            dec_once(d, x)
        asm[k] = sum(ev.device_time_total for ev in prof.key_averages() if ev.key.startswith("ragged_")) / 1e3
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    med = {k: statistics.median(v) for k, v in t.items()}
    print(json.dumps({"gpu": gpu, "records": n, "framed_bytes_lengths": len(data_len), "framed_bytes_splits": len(data),
                      "checked": True,
                      "decode_lengths_GBps": len(data_len) / med["decode_lengths"] / 1e9,
                      "decode_splits_GBps": len(data) / med["decode_splits"] / 1e9,
                      "decode_lengths_ms": med["decode_lengths"] * 1e3, "decode_splits_ms": med["decode_splits"] * 1e3,
                      "assembly_lengths_ms": asm["lengths"], "assembly_splits_ms": asm["splits"],
                      "encode_lengths_GBps": len(data_len) / med["encode_lengths"] / 1e9,
                      "encode_splits_GBps": len(data) / med["encode_splits"] / 1e9}))


if __name__ == "__main__":
    main()
