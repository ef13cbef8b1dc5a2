"""Times TFR_F_RESYNC on a configs[1] block (oracle.corpus.cfg2_columns, about 1.7 KB per record) decoded from device memory,
in one process, arms alternated round by round:
  (d0)    DROPMALFORMED without the flag, the clean block
  (r0)    DROPMALFORMED with TFR_F_RESYNC, the clean block: the pipelined path of (d0), the chains verifying every header
  (r1)    with the flag, the block with one broken header (a flipped length-CRC bit: one lost region)
  (rmib)  with the flag, one broken header per MiB
Each arm has its own decoder, warmed up on its block first, so that (d0) and (r0) run in their pipelined steady state and
(r1) / (rmib) show what a damaged block costs there: the pipelined attempt, then the synchronous resync path (a frame index
and a resync scan per region, the gather of the frames, their decode).  Checks every result's rows, entries, lost regions and
consumed bytes.  Prints the card, its power limit and max SM clock, and per arm the median, min and max of the rounds, and
the cost per lost region over (r0).

usage: python tools/quick_resync.py [BLOCK_MIB] [ROUNDS]"""
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
    block_mib = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 7
    if not torch.cuda.is_available():
        raise SystemExit("quick_resync: no CUDA device (this measurement runs on the GPU only)")
    print("card:", card(), "| torch", torch.__version__)
    n = block_mib * (1 << 20) // 1650
    sch, cols = corpus.cfg2_columns(n, seed=2024)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0 and len(data) < 1 << 31
    offs = record_offsets(data)
    clean = np.frombuffer(data, dtype=np.uint8).copy()
    blocks = {"d0": clean, "r0": clean}
    for name, k in (("r1", 1), ("rmib", max(1, len(data) >> 20))):
        b = clean.copy()
        for i in np.linspace(n // (2 * k), n - 1, k).astype(np.int64):
            b[offs[i] + 8] ^= 0x01                                # the length CRC: a framing error, one frame lost
        blocks[name] = (b, k)
    print(f"block: {len(data) / 2**20:.1f} MiB, {n} records; rounds {rounds}")
    arms, want = {}, {}
    for name, v in blocks.items():
        host, k = (v, 0) if isinstance(v, np.ndarray) else v
        flags = A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED | (0 if name == "d0" else A.TFR_F_RESYNC)
        arms[name] = (_native.Decoder(sch, 0, flags=flags), torch.from_numpy(host).cuda())
        want[name] = k
    times = {k: [] for k in arms}
    for r in range(rounds + 2):                                  # two warm-up rounds (shape learning, module loads)
        for name, (dec, dev) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b, used = dec.decode(dev)
            dt = time.perf_counter() - t0
            info, nd = b.info, len(b.dropped())
            k = want[name]
            assert used == len(data) and info["error_code"] == 0 and nd == k, (name, info, nd)
            assert info["n_rows"] == n - k and info["n_records"] == n, (name, info)
            b.release()
            if r >= 2:
                times[name].append(dt * 1e3)
    med = {}
    for name, (dec, _) in arms.items():
        t = np.array(times[name])
        med[name] = float(np.median(t))
        st = dec.stats()
        print(f"{name:5s} median {med[name]:8.2f} ms  min {t.min():8.2f}  max {t.max():8.2f}  "
              f"{len(data) / med[name] / 1e6:7.1f} GB/s   speculative {st['speculative_submits']} redone {st['speculative_redone']} "
              f"lost regions {st['lost_regions']}")
        dec.close()
    for name in ("r1", "rmib"):
        print(f"{name}: {(med[name] - med['r0']) / want[name]:.3f} ms per lost region over r0 ({want[name]} regions per block)")
    print(f"r0 / d0 (clean data, the flag's cost): {med['r0'] / med['d0']:.3f}")


if __name__ == "__main__":
    main()
