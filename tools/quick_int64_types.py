"""extendedTypes=true on one GPU.  A seeded corpus of Example records with 16 BooleanType, 16 DateType and 16 TimestampType scalars
and 8 ArrayType(BooleanType) fields (0-16 elements), built as numpy columns, is encoded once with the extended schema and once as
the same data in LongType columns.  Before any time is reported every output is checked:
  - the two encodes are byte-identical (the file bytes are those of the LongType fields with the widened values);
  - the extended decode gives back the narrow input columns, and the LongType decode the widened ones;
  - tfr_encode_rows of each decoded batch's UnsafeRows gives the same bytes again.
Then, the arms alternated rep by rep after a warm-up (medians, CUDA events around each synchronous call):
  - resident decode GB/s (device input), extended and LongType;
  - the narrow kernel's share of the extended decode (torch.profiler, a run of its own);
  - encode GB/s of framed output from host columns (tfr_encode), extended (with its widening launch) and LongType;
  - encode GB/s of framed output from host UnsafeRows (tfr_encode_rows), extended (narrow slots and elements) and LongType.
Prints one JSON line with the card's name and power limit, read in the same call."""
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
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(HERE, ".."))
    import numpy as np
    import torch
    from spark_tfrecord_b200 import _native
    from spark_tfrecord_b200 import _cabi as A
    from spark_tfrecord_b200.sqltypes import (ArrayType, BooleanType, DateType, LongType, StructField, StructType,
                                              TimestampType)

    n = a.records
    rng = np.random.default_rng(0)
    kinds = [("b", BooleanType(), A.TFR_T_BOOL)] * 16 + [("d", DateType(), A.TFR_T_DATE)] * 16 + \
            [("t", TimestampType(), A.TFR_T_TIMESTAMP)] * 16
    ext = StructType([StructField(f"{k}{i}", t, True) for i, (k, t, _) in enumerate(kinds)] +
                     [StructField(f"ab{i}", ArrayType(BooleanType()), True) for i in range(8)])
    lng = StructType([StructField(f.name, ArrayType(LongType()) if isinstance(f.dataType, ArrayType) else LongType(), True)
                      for f in ext])
    valid = np.full((n + 7) // 8, 0xFF, np.uint8)
    cols_e, cols_l = [], []
    for _, _, tid in kinds:
        v = (rng.integers(0, 2, n).astype(np.uint8) if tid == A.TFR_T_BOOL else
             rng.integers(-30000, 30000, n).astype(np.int32) if tid == A.TFR_T_DATE else
             rng.integers(-2**50, 2**50, n).astype(np.int64))
        cols_e.append(A.HostColumn(tid, 0, n, valid, [], v))
        cols_l.append(A.HostColumn(A.TFR_T_INT64, 0, n, valid, [], v.astype(np.int64)))
    for _ in range(8):
        off = np.concatenate([[0], np.cumsum(rng.integers(0, 17, n))]).astype(np.int32)
        v = rng.integers(0, 2, int(off[-1])).astype(np.uint8)
        cols_e.append(A.HostColumn(A.TFR_T_BOOL, 1, n, valid, [off], v))
        cols_l.append(A.HostColumn(A.TFR_T_INT64, 1, n, valid, [off], v.astype(np.int64)))
    enc_e = _native.Encoder(ext, 0, extended_types=True)
    enc_l = _native.Encoder(lng, 0)
    data = enc_e.encode(cols_e)
    # ---- checks ----
    assert enc_l.encode(cols_l) == data, "the extended encode differs from the LongType encode of the widened values"
    dev = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    dec_e = _native.Decoder(ext, 0, extended_types=True)
    dec_l = _native.Decoder(lng, 0)
    urows = {}
    for d, cols, enc in ((dec_e, cols_e, enc_e), (dec_l, cols_l, enc_l)):
        b, _ = d.decode(dev)
        assert b.info["error_code"] == 0 and b.n_rows == n
        for c, g in zip(cols, b.to_host()):
            assert g.elem_type == c.elem_type and np.array_equal(g.values, c.values)
            assert all(np.array_equal(o, go) for o, go in zip(c.offsets, g.offsets))
        rows, offs = b.unsafe_rows()
        urows[id(enc)] = (rows.copy(), offs.astype(np.int32))
        b.release()
        enc.encode_rows(*urows[id(enc)])
        assert enc.result_host() == data, "the UnsafeRows encode differs from the columns encode"
    rows_e, rows_l = urows[id(enc_e)], urows[id(enc_l)]

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

    arms = {"decode_ext": lambda: dec_once(dec_e), "decode_long": lambda: dec_once(dec_l),
            "encode_ext": lambda: enc_e.encode(cols_e), "encode_long": lambda: enc_l.encode(cols_l),
            "rows_ext": lambda: enc_e.encode_rows(*rows_e), "rows_long": lambda: enc_l.encode_rows(*rows_l)}
    for f in arms.values():
        f(); f()
    t = {k: [] for k in arms}
    for _ in range(a.reps):
        for k, f in arms.items():
            t[k].append(timed(f))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dec_once(dec_e)
    nar = sum(ev.device_time_total for ev in prof.key_averages() if "narrow_kernel" in ev.key) / 1e3
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    med = {k: statistics.median(v) for k, v in t.items()}
    print(json.dumps({"gpu": gpu, "records": n, "framed_bytes": len(data), "checked": True,
                      "decode_ext_GBps": len(data) / med["decode_ext"] / 1e9,
                      "decode_long_GBps": len(data) / med["decode_long"] / 1e9,
                      "narrow_ms": nar, "decode_ext_ms": med["decode_ext"] * 1e3,
                      "encode_ext_GBps": len(data) / med["encode_ext"] / 1e9,
                      "encode_long_GBps": len(data) / med["encode_long"] / 1e9,
                      "encode_rows_ext_GBps": len(data) / med["rows_ext"] / 1e9,
                      "encode_rows_long_GBps": len(data) / med["rows_long"] / 1e9,
                      "rows_bytes_ext": int(rows_e[1][-1]), "rows_bytes_long": int(rows_l[1][-1])}))


if __name__ == "__main__":
    main()
