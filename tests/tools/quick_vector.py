"""VectorUDT against ArrayType(DoubleType) on one GPU, the two alternated rep by rep, median seconds and GB/s of row input:
  encode_dense128 : tfr_encode_rows of 1 M rows of 128-d dense vectors, and of the same values as ArrayType(DoubleType) rows;
  encode_sparse   : 50 k sparse rows of size 4,096 with 64 non-zeros, and the same values densified as double-array rows;
  rows_dense128   : tfr_batch_rows (device) of the decoded vector column, and of the ArrayType(DoubleType) column.
Rows are device-resident (the encoder's input) and built with numpy.  Prints one JSON line per workload with the card's name
and power limit, read in the same call."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))

import numpy as np


def _arr_bytes(n, esz):
    return 8 + 8 * ((n + 63) // 64) + (n * esz + 7) // 8 * 8


def double_rows(vals):
    """rows (id: long, v: array<double>) of a [n, k] float64 matrix -> (uint8 rows, int32 offsets)"""
    n, k = vals.shape
    ab = _arr_bytes(k, 8)
    size = 8 + 16 + ab
    R = np.zeros((n, size), np.uint8)
    R[:, 8:16].view(np.int64)[:, 0] = np.arange(n)
    R[:, 16:24].view(np.uint64)[:, 0] = np.uint64((24 << 32) | ab)
    R[:, 24:32].view(np.int64)[:, 0] = k
    R[:, size - k * 8:].view(np.float64)[:] = vals
    return R.reshape(-1), (np.arange(n + 1, dtype=np.int64) * size).astype(np.int32)


def dense_vector_rows(vals):
    """rows (id: long, v: VectorUDT) of dense vectors: the nested struct of include/tfrgpu.h, VECTORS"""
    n, k = vals.shape
    ab = _arr_bytes(k, 8)
    size = 8 + 16 + 40 + ab
    R = np.zeros((n, size), np.uint8)
    W = R[:, :64].view(np.uint64)
    W[:, 1] = np.arange(n, dtype=np.uint64)
    W[:, 2] = np.uint64((24 << 32) | (40 + ab))
    W[:, 3] = 6                                    # the nested row: size and indices null
    W[:, 4] = 1                                    # type dense
    W[:, 7] = np.uint64((40 << 32) | ab)
    R[:, 64:72].view(np.int64)[:, 0] = k
    R[:, size - k * 8:].view(np.float64)[:] = vals
    return R.reshape(-1), (np.arange(n + 1, dtype=np.int64) * size).astype(np.int32)


def sparse_vector_rows(size, idx, vals):
    """rows (id: long, v: VectorUDT) of sparse vectors of `size`, idx / vals [n, nnz]"""
    n, m = idx.shape
    ib, vb = _arr_bytes(m, 4), _arr_bytes(m, 8)
    rs = 8 + 16 + 40 + ib + vb
    R = np.zeros((n, rs), np.uint8)
    W = R[:, :64].view(np.uint64)
    W[:, 1] = np.arange(n, dtype=np.uint64)
    W[:, 2] = np.uint64((24 << 32) | (40 + ib + vb))
    W[:, 4] = 0
    W[:, 5] = size
    W[:, 6] = np.uint64((40 << 32) | ib)
    W[:, 7] = np.uint64(((40 + ib) << 32) | vb)
    R[:, 64:72].view(np.int64)[:, 0] = m
    R[:, 64 + ib - (4 * m + 7) // 8 * 8:64 + ib - (4 * m + 7) // 8 * 8 + 4 * m].view(np.int32)[:] = idx
    R[:, 64 + ib:72 + ib].view(np.int64)[:, 0] = m
    R[:, rs - 8 * m:].view(np.float64)[:] = vals
    return R.reshape(-1), (np.arange(n + 1, dtype=np.int64) * rs).astype(np.int32)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--rows", type=int, default=1_000_000)
    a = ap.parse_args()
    import torch
    from spark_tfrecord_b200 import _native
    from spark_tfrecord_b200.sqltypes import ArrayType, DoubleType, LongType, StructField, StructType, VectorUDT
    sv = StructType([StructField("id", LongType()), StructField("v", VectorUDT())])
    sd = StructType([StructField("id", LongType()), StructField("v", ArrayType(DoubleType()))])
    rng = np.random.default_rng(0)
    info = gpu_info()

    def encoder_arm(sch, rows):
        dr, do = torch.from_numpy(rows[0]).cuda(), torch.from_numpy(rows[1]).cuda()
        enc = _native.Encoder(sch)
        for _ in range(2):
            enc.encode_rows(dr, do)
        out = enc.result_host()
        return enc, (lambda: enc.encode_rows(dr, do)), out, rows[0].nbytes

    vals = rng.standard_normal((a.rows, 128)).astype(np.float32).astype(np.float64)
    sn = max(a.rows // 20, 1000)
    idx = np.sort(np.argsort(rng.random((sn, 4096)), axis=1)[:, :64], axis=1).astype(np.int32)
    sval = rng.standard_normal((sn, 64)).astype(np.float32).astype(np.float64)
    dense_of_sparse = np.zeros((sn, 4096))
    np.put_along_axis(dense_of_sparse, idx, sval, axis=1)
    workloads = {"encode_dense128": ((sv, dense_vector_rows(vals)), (sd, double_rows(vals))),
                 "encode_sparse": ((sv, sparse_vector_rows(4096, idx, sval)), (sd, double_rows(dense_of_sparse)))}
    for name, ((s1, r1), (s2, r2)) in workloads.items():
        e1, f1, o1, b1 = encoder_arm(s1, r1)
        e2, f2, o2, b2 = encoder_arm(s2, r2)
        assert o1 == o2, f"{name}: the vector rows' bytes differ from the double rows'"
        t1, t2 = [], []
        for _ in range(a.reps):                        # alternated
            t1 += timed(f1, 1)
            t2 += timed(f2, 1)
        e1.close(); e2.close()
        m1, m2 = statistics.median(t1), statistics.median(t2)
        print(json.dumps({"workload": name, "gpu": info, "vector_s": m1, "double_s": m2, "vector_over_double": m1 / m2,
                          "vector_in_GBps": b1 / m1 / 1e9, "double_in_GBps": b2 / m2 / 1e9, "out_bytes": len(o1)}), flush=True)
        del e1, e2
        if name == "encode_dense128":
            framed = o1
    # rows of a decoded batch
    dev = torch.frombuffer(bytearray(framed), dtype=torch.uint8).cuda()
    decs = {"vector": _native.Decoder(sv), "double": _native.Decoder(sd)}
    ts = {k: [] for k in decs}
    nbytes = {}
    for rep in range(a.reps + 1):
        for k, dec in decs.items():
            b, _ = dec.decode(dev)
            b.wait()
            t = timed(lambda: b.unsafe_rows(to_host=False), 1)
            nbytes[k] = b.unsafe_rows(to_host=False)[3]
            b.release()
            if rep:
                ts[k] += t
    mv, md = statistics.median(ts["vector"]), statistics.median(ts["double"])
    print(json.dumps({"workload": "rows_dense128", "gpu": info, "vector_s": mv, "double_s": md, "vector_over_double": mv / md,
                      "vector_rows_GBps": nbytes["vector"] / mv / 1e9, "double_rows_GBps": nbytes["double"] / md / 1e9}), flush=True)
    for d in decs.values():
        d.close()


if __name__ == "__main__":
    main()
