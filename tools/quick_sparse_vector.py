"""The sparse vector format (vectorFormat=sparse) against the dense one on one GPU, the two arms alternated rep by rep after a
warm-up, median seconds.  Workloads (rows (id: long, v: VectorUDT), device-resident, built with numpy):
  tf4096   : 200 k rows of size 4,096 with 64 non-zeros; the dense arm runs in calls of 50 k rows (its densify limit);
  hash2e18 : 4 k rows of size 2^18 with 64 non-zeros (HashingTF-like); the dense arm runs in calls of 1,024 rows, because
             2,048 or more reach its densify limit.
For each: the framed output bytes, tfr_encode_rows time, and decode (device input) + tfr_batch_rows (device) time.
--rows-only: only tfr_batch_rows of 1 M decoded 128-d dense vectors (UR_VEC rows), for a before / after comparison of that
path; --root picks the tree to import the package from.  Prints one JSON line per figure with the card's name, power limit and
max SM clock, read in the same call."""
import argparse
import json
import os
import statistics
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rows-only", action="store_true")
    ap.add_argument("--root", default=os.path.join(HERE, ".."))
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.root))
    sys.path.insert(0, os.path.join(HERE, "..", "tests", "tools"))
    import numpy as np
    import torch
    from quick_vector import dense_vector_rows, gpu_info, sparse_vector_rows, timed
    from spark_tfrecord_b200 import _native
    from spark_tfrecord_b200.sqltypes import LongType, StructField, StructType, VectorUDT
    sch = StructType([StructField("id", LongType()), StructField("v", VectorUDT())])
    info = gpu_info()
    rng = np.random.default_rng(0)

    def rows_time(dec, dev):
        b, _ = dec.decode(dev)
        b.wait()
        t = timed(lambda: b.unsafe_rows(to_host=False), 1)
        b.release()
        return t

    if a.rows_only:
        vals = rng.standard_normal((1_000_000, 128)).astype(np.float32).astype(np.float64)
        dr, do = (torch.from_numpy(x).cuda() for x in dense_vector_rows(vals))
        enc = _native.Encoder(sch)
        enc.encode_rows(dr, do)
        dev = torch.frombuffer(bytearray(enc.result_host()), dtype=torch.uint8).cuda()
        enc.close()
        dec = _native.Decoder(sch)
        rows_time(dec, dev)
        ts = [t for _ in range(a.reps) for t in rows_time(dec, dev)]
        dec.close()
        print(json.dumps({"workload": "rows_dense128_urvec", "root": os.path.abspath(a.root), "gpu": info,
                          "batch_rows_s": statistics.median(ts)}), flush=True)
        return

    for name, n, size, chunk in (("tf4096", 200_000, 4096, 50_000), ("hash2e18", 4096, 1 << 18, 1024)):
        idx = np.sort(np.stack([rng.choice(size, 64, replace=False) for _ in range(n)]), axis=1).astype(np.int32)
        val = rng.standard_normal((n, 64)).astype(np.float32).astype(np.float64)
        arms = {}
        for vf in ("sparse", "dense"):
            step = n if vf == "sparse" else chunk
            calls = []
            for s in range(0, n, step):
                r, o = sparse_vector_rows(size, idx[s:s + step], val[s:s + step])
                calls.append((torch.from_numpy(r).cuda(), torch.from_numpy(o).cuda()))
            enc = _native.Encoder(sch, vector_format=vf)
            dec = _native.Decoder(sch, vector_format=vf)
            out = []
            for dr, do in calls:                                  # warm-up, and the framed output
                enc.encode_rows(dr, do)
                out.append(enc.result_host())
            devs = [torch.frombuffer(bytearray(o), dtype=torch.uint8).cuda() for o in out]
            for d in devs:
                rows_time(dec, d)
            arms[vf] = dict(enc=enc, dec=dec, calls=calls, devs=devs, out_bytes=sum(len(o) for o in out), te=[], tr=[])

        def encode_all(A):
            for dr, do in A["calls"]:
                A["enc"].encode_rows(dr, do)

        def decode_rows_all(A):
            for d in A["devs"]:
                b, _ = A["dec"].decode(d)
                b.unsafe_rows(to_host=False)
                b.release()
        for _ in range(a.reps):                                   # alternated
            for A in arms.values():
                A["te"] += timed(lambda: encode_all(A), 1)
                A["tr"] += timed(lambda: decode_rows_all(A), 1)
        res = {"workload": name, "rows": n, "size": size, "nnz": 64, "dense_call_rows": chunk, "gpu": info}
        for vf, A in arms.items():
            res[vf + "_out_bytes"] = A["out_bytes"]
            res[vf + "_encode_rows_s"] = statistics.median(A["te"])
            res[vf + "_decode_and_rows_s"] = statistics.median(A["tr"])
            A["enc"].close()
            A["dec"].close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
