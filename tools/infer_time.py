"""infer_kernel time on one large corpus, for comparing two builds of the library in one run.

    python tools/infer_time.py [--records 1000000] [--rounds 2] [--record-type 0|1] [--mode FAILFAST|DROPMALFORMED|PERMISSIVE]
                               [--bad-every K] [--seed S] [LIB.so | TREE ...]

Encodes `--records` configs[1] records (oracle/corpus.cfg2_columns; as SequenceExamples with --record-type 1) once into a
temporary file, then, for each round, runs every library (default: the tree's own build) in a fresh process, alternating
them.  A LIB.so is loaded by this tree's bindings; a TREE (a directory holding another checkout and its build) is
imported whole, for builds whose C ABI this tree's bindings do not match.  Each process puts the whole batch on the
device, infers in `--mode` (PERMISSIVE with the corrupt-record column _corrupt_record), warms up with one `Infer.update`,
then profiles three more and reports the mean `infer_kernel` device time (torch.profiler, CUDA activities), the mean wall
time of an update and the records skipped.  With `--bad-every K` every K-th record is damaged, a flipped data CRC or an
entry whose kind is not set, chosen from `--seed`.  One JSON line per process."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


MODES = {"FAILFAST": (0, None), "DROPMALFORMED": (0x3, None), "PERMISSIVE": (0x5, "_corrupt_record")}


def damage(data: bytes, k: int, seed: int) -> bytes:
    """every k-th record: its data CRC flipped, or an entry whose kind is not set put in front of its payload (re-framed)"""
    import random
    import struct
    from oracle import oracle
    R = random.Random(seed)
    out, pos, row = [], 0, 0
    while pos < len(data):
        n = struct.unpack_from("<Q", data, pos)[0]
        frame = data[pos:pos + 16 + n]
        if row % k == k - 1:
            if R.random() < 0.5:
                frame = frame[:-1] + bytes([frame[-1] ^ 0x10])
            else:
                payload = b"\x0a\x08\x0a\x06\x0a\x02_b\x12\x00" + frame[12:-4]      # features/context {"_b": Feature()}
                hdr = struct.pack("<Q", len(payload))
                frame = hdr + struct.pack("<I", oracle.masked_crc32c(hdr)) + payload + struct.pack("<I", oracle.masked_crc32c(payload))
        out.append(frame)
        pos += 16 + n
        row += 1
    return b"".join(out)


def child(path, n, rt, mode):
    sys.path.insert(0, os.environ.get("INFER_TIME_TREE") or ROOT)
    import time
    import numpy as np
    import torch
    from spark_tfrecord_b200 import _native
    data = torch.from_numpy(np.fromfile(path, np.uint8)).cuda()
    flags, name = MODES[mode]
    inf = _native.Infer(rt, 0, flags, name) if mode != "FAILFAST" else _native.Infer(rt)
    inf.update(data)
    want = inf.result()
    skipped = len(inf.skipped()) if mode != "FAILFAST" else 0
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
    ks = [e for e in prof.events() if "infer_kernel" in e.name]            # (infer_kernel<false> / <true> are templates)
    dev = [getattr(e, "device_time", None) or e.cuda_time for e in ks]
    print(json.dumps({"lib": os.environ.get("INFER_TIME_TREE") or os.environ.get("TFR_LIB", "tree"), "records": n,
                      "record_type": rt, "mode": mode, "skipped": skipped, "bytes": int(data.numel()),
                      "infer_kernel_ms": round(sum(dev) / len(dev) / 1e3, 3), "kernels": len(dev),
                      "update_wall_ms": round(1e3 * sum(walls) / len(walls), 3), "names": len(want)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--record-type", type=int, default=0, choices=[0, 1])
    ap.add_argument("--mode", default="FAILFAST", choices=sorted(MODES))
    ap.add_argument("--bad-every", type=int, default=0)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--child", default=None)
    ap.add_argument("libs", nargs="*")
    a = ap.parse_args()
    if a.child:
        return child(a.child, a.records, a.record_type, a.mode)
    sys.path.insert(0, ROOT)
    from oracle import corpus, oracle
    sch, cols = corpus.cfg2_columns(a.records, seed=2)
    data, rc, _ = oracle.encode(cols, sch, a.record_type)
    assert rc == 0
    if a.bad_every:
        data = damage(data, a.bad_every, a.seed)
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
                if lib and os.path.isdir(lib):
                    env["INFER_TIME_TREE"] = os.path.abspath(lib)
                elif lib:
                    env["TFR_LIB"] = os.path.abspath(lib)
                subprocess.run([sys.executable, os.path.abspath(__file__), "--child", path, "--records", str(a.records),
                                "--record-type", str(a.record_type), "--mode", a.mode], env=env, check=True)


if __name__ == "__main__":
    main()
