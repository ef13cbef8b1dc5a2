"""Record index measurements (include/tfrgpu.h, RECORD INDEX) on one GPU, printed as one JSON line:

  - build rate: tfr_index_update over a configs[1] file in one final block, from device memory and from pinned host memory
    (the host case includes the H2D copy), median of several runs, GB/s of data indexed;
  - the writer's extra time per flush with recordIndex=true: the index update on the encoder's device result of one
    65,536-row configs[1] flush, against the flush's encode + host copy;
  - the bytes a split read touches beyond its range: the two seeks' bytes plus the frames read past the split's end, over
    128 MiB splits of the file at the writer's stride (1 MiB).

Usage: python tools/quick_record_index.py [--records N] [--reps R]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import corpus, oracle  # noqa: E402
from spark_tfrecord_b200 import _native  # noqa: E402
from spark_tfrecord_b200 import io as tio  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=400_000)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these numbers are only measured on the GPU")
    schema, cols = corpus.cfg2_columns(a.records, seed=3)
    data, rc, _ = oracle.encode(cols, schema)
    assert rc == 0
    data = bytes(data)
    stride = tio.RECORD_INDEX_STRIDE
    host = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).pin_memory()
    dev = host.cuda()
    torch.cuda.synchronize()
    res = {"gpu": gpu_info(), "file_bytes": len(data), "records": a.records, "stride": stride}

    ref = None
    for name, src in (("device", dev), ("pinned_host", (host.data_ptr(), len(data), 0))):
        def run():
            idx = _native.Indexer(stride)
            try:
                idx.update(src, True)
                return idx.result()
            finally:
                idx.close()
        got = run()                                                  # warm-up, and the result every arm must give
        ref = ref or got
        assert got == ref
        t = timed(run, a.reps)
        res[f"build_{name}_ms"] = round(t * 1e3, 3)
        res[f"build_{name}_GBps"] = round(len(data) / t / 1e9, 2)

    # the writer's flush: encode + host copy, then the index update on the encoder's device bytes
    fs, fcols = corpus.cfg2_columns(65536, seed=4)
    enc = _native.Encoder(fs)
    ctc = [c.to_ctypes() for c in fcols]
    idx = _native.Indexer(stride)

    def flush(indexed):
        ptr, n = enc.encode_columns(ctc, False)
        enc.result_host()
        if indexed:
            t0 = time.perf_counter()
            idx.update((ptr, n, 1), False)
            return time.perf_counter() - t0
        return 0.0

    flush(True)
    plain, extra = [], []
    for _ in range(a.reps):                                         # the two arms alternated
        t0 = time.perf_counter(); flush(False); plain.append(time.perf_counter() - t0)
        extra.append(flush(True))
    idx.close()
    enc.close()
    res["flush_encode_ms"] = round(float(np.median(plain)) * 1e3, 3)
    res["flush_index_extra_ms"] = round(float(np.median(extra)) * 1e3, 3)

    # the bytes a split read touches beyond its range
    n_entries, _, ck = tio.parse_index(ref, len(data))
    seeker = _native.Indexer(stride)
    split = 128 << 20
    over, splits = [], 0
    for s in range(0, len(data), split):
        e = min(len(data), s + split)
        touched = 0
        bounds = []
        for t in (s, e):
            if t >= len(data):
                bounds.append(len(data))
                continue
            off, ent = int(ck[t // stride][0]), int(ck[t // stride][1])
            nb = max(0, min(len(data), t + 12) - off)
            touched += nb
            bounds.append(seeker.seek(data[off:off + nb], ent, off, t)[1])
        touched += bounds[1] - bounds[0]
        over.append(touched - (e - s))
        splits += 1
    seeker.close()
    res["split_bytes"] = split
    res["splits"] = splits
    res["split_extra_bytes_max"] = int(max(over))
    res["split_extra_bytes_mean"] = round(float(np.mean(over)), 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
