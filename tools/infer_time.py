"""infer_kernel time on one large corpus, for comparing two builds of the library in one run.

    python tools/infer_time.py [--records 1000000] [--rounds 2] [LIB.so ...]

Encodes `--records` configs[1] records (oracle/corpus.cfg2_columns) once into a temporary file, then, for each round,
runs every library (default: the tree's own build) in a fresh process, alternating them.  Each process puts the whole
batch on the device, warms up with one `Infer.update`, then profiles three more and reports the mean `infer_kernel`
device time (torch.profiler, CUDA activities) and the mean wall time of an update.  One JSON line per process."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child(path, n):
    sys.path.insert(0, ROOT)
    import time
    import numpy as np
    import torch
    from spark_tfrecord_b200 import _native
    data = torch.from_numpy(np.fromfile(path, np.uint8)).cuda()
    inf = _native.Infer(0)
    inf.update(data)
    want = inf.result()
    walls = []
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            torch.cuda.synchronize()
            t = time.perf_counter()
            inf.update(data)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t)
    assert inf.result() == want
    inf.close()
    ks = [e for e in prof.events() if e.name.startswith("infer_kernel")]
    dev = [getattr(e, "device_time", None) or e.cuda_time for e in ks]
    print(json.dumps({"lib": os.environ.get("TFR_LIB", "tree"), "records": n, "bytes": int(data.numel()),
                      "infer_kernel_ms": round(sum(dev) / len(dev) / 1e3, 3), "kernels": len(dev),
                      "update_wall_ms": round(1e3 * sum(walls) / len(walls), 3), "names": len(want)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--child", default=None)
    ap.add_argument("libs", nargs="*")
    a = ap.parse_args()
    if a.child:
        return child(a.child, a.records)
    sys.path.insert(0, ROOT)
    from oracle import corpus, oracle
    sch, cols = corpus.cfg2_columns(a.records, seed=2)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip()}), flush=True)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "cfg2.tfrecord")
        with open(path, "wb") as f:
            f.write(data)
        del data, cols
        libs = a.libs or [None]
        for _ in range(a.rounds):
            for lib in libs:
                env = dict(os.environ)
                if lib:
                    env["TFR_LIB"] = os.path.abspath(lib)
                subprocess.run([sys.executable, os.path.abspath(__file__), "--child", path, "--records", str(a.records)],
                               env=env, check=True)


if __name__ == "__main__":
    main()
