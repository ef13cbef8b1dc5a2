"""Times PERMISSIVE (TFR_F_PERMISSIVE) against FAILFAST and drop mode on a configs[1] block (oracle.corpus.cfg2_columns,
about 1.7 KB per record) decoded from device memory, in one process, arms alternated round by round:
  (ff)     FAILFAST (the default flags), the clean block
  (p0)     PERMISSIVE with a corrupt-record column (appended to the schema), the clean block
  (p0n)    PERMISSIVE without a corrupt-record column, the clean block
  (p1)     PERMISSIVE with the column, the block with 1 bad record (a payload bit flip: a data CRC mismatch)
  (p1000)  PERMISSIVE with the column, the block with 1,000 bad records, evenly spread
  (d1)     drop mode, the block with 1 bad record
  (d1000)  drop mode, the block with 1,000 bad records
Each arm has its own decoder, warmed up on its block first, so that the clean arms run in their pipelined steady state and
the bad ones show what a bad block costs there.  Checks every result's row count, corrupt or dropped count and consumed
bytes.  Every arm is timed from a synchronised device to the end of all the batch's device work (tfr_decode returns
before the last kernels of a PERMISSIVE bad block have run).  Prints the card, its power limit and max SM clock, and per
arm the median, min and max of the rounds.

usage: python tools/quick_permissive.py [BLOCK_MIB] [ROUNDS]"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import corpus, oracle  # noqa: E402
from quick_drop import card  # noqa: E402
from spark_tfrecord_b200 import _cabi as A  # noqa: E402
from spark_tfrecord_b200 import _native  # noqa: E402
from spark_tfrecord_b200.sqltypes import BinaryType, StructField, StructType  # noqa: E402
from util import record_offsets  # noqa: E402

PERM = A.TFR_F_DEFAULT | A.TFR_F_PERMISSIVE
DROP = A.TFR_F_DEFAULT | A.TFR_F_DROP_MALFORMED


def main():
    block_mib = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 9
    if not torch.cuda.is_available():
        raise SystemExit("quick_permissive: no CUDA device (this measurement runs on the GPU only)")
    print("card:", card(), "| torch", torch.__version__)
    n = block_mib * (1 << 20) // 1650
    sch, cols = corpus.cfg2_columns(n, seed=2024)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0
    while len(data) >= 1 << 31:                                 # a block stays below 2 GiB
        n = n * 15 // 16
        sch, cols = corpus.cfg2_columns(n, seed=2024)
        data, rc, _ = oracle.encode(cols, sch)
    full = StructType(list(sch.fields) + [StructField("_corrupt_record", BinaryType())])
    cf = len(sch.fields)
    offs = record_offsets(data)
    clean = np.frombuffer(data, dtype=np.uint8).copy()
    dev = {"clean": torch.from_numpy(clean).cuda()}
    for k in (1, 1000):
        b = clean.copy()
        for i in np.linspace(n // (2 * k), n - 1, k).astype(np.int64):
            b[offs[i] + 12] ^= 0x01                               # first payload byte: the data CRC no longer matches
        dev[k] = torch.from_numpy(b).cuda()
    print(f"block: {len(data) / 2**20:.1f} MiB, {n} records; rounds {rounds}")
    # name: (decoder, block, bad records expected, rows expected)
    arms = {
        "ff": (_native.Decoder(sch, 0, flags=A.TFR_F_DEFAULT), dev["clean"], 0, n),
        "p0": (_native.Decoder(full, 0, flags=PERM, corrupt_field=cf), dev["clean"], 0, n),
        "p0n": (_native.Decoder(sch, 0, flags=PERM), dev["clean"], 0, n),
        "p1": (_native.Decoder(full, 0, flags=PERM, corrupt_field=cf), dev[1], 1, n),
        "p1000": (_native.Decoder(full, 0, flags=PERM, corrupt_field=cf), dev[1000], 1000, n),
        "d1": (_native.Decoder(sch, 0, flags=DROP), dev[1], 1, n - 1),
        "d1000": (_native.Decoder(sch, 0, flags=DROP), dev[1000], 1000, n - 1000),
    }
    times = {k: [] for k in arms}
    for r in range(rounds + 2):                                  # two warm-up rounds (shape learning, module loads)
        for name, (dec, block, n_bad, n_rows) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b, used = dec.decode(block)
            torch.cuda.synchronize()                             # tfr_decode returns with the last kernels still queued
            dt = time.perf_counter() - t0
            info, nb = b.info, len(b.dropped())
            assert used == len(data) and info["error_code"] == 0 and nb == n_bad, (name, info, nb)
            assert info["n_rows"] == n_rows and info["n_records"] == n, (name, info)
            b.release()
            if r >= 2:
                times[name].append(dt * 1e3)
    for name, (dec, *_) in arms.items():
        t = np.array(times[name])
        st = dec.stats()
        print(f"{name:6s} median {np.median(t):8.2f} ms  min {t.min():8.2f}  max {t.max():8.2f}  "
              f"{len(data) / np.median(t) / 1e6:7.1f} GB/s   speculative {st['speculative_submits']} redone {st['speculative_redone']} "
              f"corrupt {st['records_corrupt']} dropped {st['records_dropped']}")
        dec.close()


if __name__ == "__main__":
    main()
