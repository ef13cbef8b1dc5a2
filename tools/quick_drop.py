"""Times drop mode (TFR_F_DROP_MALFORMED) on a configs[1] block (oracle.corpus.cfg2_columns, about 1.7 KB per record)
decoded from device memory, in one process, arms alternated round by round:
  (ff)    FAILFAST (the default flags), the clean block
  (d0)    drop mode, the clean block: the same path as (ff)
  (d1)    drop mode, the block with 1 bad record (a payload bit flip: a data CRC mismatch)
  (d1000) drop mode, the block with 1,000 bad records, evenly spread
  (ff1)   FAILFAST, the block with 1 bad record: the redo every such block already costs, rows up to the bad record
Each arm has its own decoder, warmed up on its block first, so that (ff) and (d0) run in their pipelined steady state and
(d1) / (d1000) show what a bad block costs there: the pipelined attempt, the general path's pass 1, the list of failing
records, the gather of the kept frames and the second decode.  Checks every result's row count, dropped count and consumed
bytes.  Prints the card, its power limit and max SM clock, and per arm the median, min and max of the rounds.

usage: python tools/quick_drop.py [BLOCK_MIB] [ROUNDS]"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import corpus, oracle  # noqa: E402
from spark_tfrecord_b200 import _cabi as A  # noqa: E402
from spark_tfrecord_b200 import _native  # noqa: E402
from util import record_offsets  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def main():
    block_mib = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 7
    if not torch.cuda.is_available():
        raise SystemExit("quick_drop: no CUDA device (this measurement runs on the GPU only)")
    print("card:", card(), "| torch", torch.__version__)
    n = block_mib * (1 << 20) // 1650
    sch, cols = corpus.cfg2_columns(n, seed=2024)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0
    while len(data) >= 1 << 31:                                 # a block stays below 2 GiB
        n = n * 15 // 16
        sch, cols = corpus.cfg2_columns(n, seed=2024)
        data, rc, _ = oracle.encode(cols, sch)
    offs = record_offsets(data)
    clean = np.frombuffer(data, dtype=np.uint8).copy()
    blocks = {"ff": clean, "d0": clean}
    for k in (1, 1000):
        b = clean.copy()
        for i in np.linspace(n // (2 * k), n - 1, k).astype(np.int64):
            b[offs[i] + 12] ^= 0x01                               # first payload byte: the data CRC no longer matches
        blocks[f"d{k}"] = b
    blocks["ff1"] = blocks["d1"]
    print(f"block: {len(data) / 2**20:.1f} MiB, {n} records; rounds {rounds}")
    arms = {}
    for name, host in blocks.items():
        flags = A.TFR_F_DEFAULT if name.startswith("ff") else A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED
        arms[name] = (_native.Decoder(sch, 0, flags=flags), torch.from_numpy(host).cuda())
    want_drop = {"ff": 0, "d0": 0, "d1": 1, "d1000": 1000, "ff1": 0}
    times = {k: [] for k in arms}
    for r in range(rounds + 2):                                  # two warm-up rounds (shape learning, module loads)
        for name, (dec, dev) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b, used = dec.decode(dev)
            dt = time.perf_counter() - t0
            info, nd = b.info, len(b.dropped())
            if name == "ff1":                                    # FAILFAST stops at the bad record
                assert info["error_code"] == A.TFR_E_CRC_DATA and info["n_rows"] == info["error_row"] and nd == 0, (name, info)
            else:
                assert used == len(data) and info["error_code"] == 0 and nd == want_drop[name], (name, info, nd)
                assert info["n_rows"] == n - nd and info["n_records"] == n, (name, info)
            b.release()
            if r >= 2:
                times[name].append(dt * 1e3)
    for name, (dec, _) in arms.items():
        t = np.array(times[name])
        st = dec.stats()
        print(f"{name:6s} median {np.median(t):8.2f} ms  min {t.min():8.2f}  max {t.max():8.2f}  "
              f"{len(data) / np.median(t) / 1e6:7.1f} GB/s   speculative {st['speculative_submits']} redone {st['speculative_redone']} "
              f"dropped {st['records_dropped']}")
        dec.close()


if __name__ == "__main__":
    main()
