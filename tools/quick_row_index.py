"""Times the generated fields (TFR_T_ROW_INDEX + TFR_T_RECORD_OFFSET, position_kernel) on resident configs[1] blocks
(oracle.corpus.cfg2_columns, about 1.7 KB per record), in one process, the two arms alternated round by round:
  (plain)  the pipelined decode of the configs[1] schema
  (gen)    the same schema with both generated fields appended, submitted at a nonzero file position
Each arm has its own decoder, warmed up first, so both run in their pipelined steady state.  A round submits K blocks back to
back from device memory and waits for the last; it is timed with CUDA events recorded on the decoder's decode stream, before
the first submit and after the last wait.  Every result is checked: rows, the data columns bit-identical between the arms,
the generated columns exact.  Then, in a pass of its own under torch.profiler, the kernels' device time per batch: the
position kernel's and the tile kernel's.  Prints the card, its power limit and max SM clock, per arm the median, min and max
ms per batch, the stats counters [1] (pipelined submits) and [2] (redone), and the position kernel's bytes per ms.

usage: python tools/quick_row_index.py [BLOCK_MIB] [ROUNDS] [K]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import corpus, oracle  # noqa: E402
from spark_tfrecord_b200 import _native  # noqa: E402
from spark_tfrecord_b200.sqltypes import RecordOffsetType, RowIndexType, StructField, StructType  # noqa: E402
from util import assert_columns_equal, record_offsets  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def main():
    block_mib = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 9
    k = int(sys.argv[3]) if len(sys.argv) > 3 else 8
    if not torch.cuda.is_available():
        raise SystemExit("quick_row_index: no CUDA device (this measurement runs on the GPU only)")
    print("card:", card(), "| torch", torch.__version__)
    n = block_mib * (1 << 20) // 1700
    sch, cols = corpus.cfg2_columns(n, seed=2024)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0 and len(data) < 1 << 31
    offs = record_offsets(data)[:-1].astype(np.int64)
    dev = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    gsch = StructType(list(sch.fields) + [StructField("_tmp_metadata_row_index", RowIndexType(), False),
                                          StructField("_tmp_metadata_record_offset", RecordOffsetType(), False)])
    nf = len(sch.fields)
    base = (5_000_000, 3 << 32)
    print(f"block: {len(data) / 2**20:.1f} MiB, {n} records ({len(data) / n:.0f} B each); rounds {rounds} x {k} blocks per arm")
    arms = {"plain": _native.Decoder(sch), "gen": _native.Decoder(gsch)}
    ref = None

    def run(name, check):
        nonlocal ref
        dec = arms[name]
        kw = {"first_entry": base[0], "first_offset": base[1]} if name == "gen" else {}
        st = torch.cuda.ExternalStream(dec.stream())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(st)
        batches = [dec.submit(dev, **kw) for _ in range(k)]
        for b in batches:
            b.wait()
        e1.record(st)
        e1.synchronize()
        for b in batches:
            assert b.n_rows == n and b.info["error_code"] == 0, (name, b.info)
        if check:
            got = batches[-1].to_host()
            if ref is None:
                ref = arms["plain"].decode(dev)[0].to_host()
            assert_columns_equal(got[:nf], ref, None, f"{name} data columns")
            if name == "gen":
                assert np.array_equal(got[nf].values, base[0] + np.arange(n)) and got[nf].null_count == 0
                assert np.array_equal(got[nf + 1].values, base[1] + offs) and got[nf + 1].null_count == 0
        for b in batches:
            b.release()
        return e0.elapsed_time(e1) / k

    for name in arms:                                    # learning, module loads, the checks
        for _ in range(4):
            run(name, True)
    s0 = {name: dec.stats() for name, dec in arms.items()}
    times = {name: [] for name in arms}
    for r in range(rounds):
        for name in (arms if r % 2 == 0 else reversed(list(arms))):
            times[name].append(run(name, r == rounds - 1))
    med = {}
    for name, dec in arms.items():
        t = np.array(times[name])
        med[name] = float(np.median(t))
        s1 = dec.stats()
        d = {key: s1[key] - s0[name][key] for key in ("batches", "speculative_submits", "speculative_redone")}
        print(f"  {name:6s} ms/batch median {med[name]:.3f}  min {t.min():.3f}  max {t.max():.3f}  "
              f"(GB/s of framed input {len(data) / med[name] / 1e6:.0f})  stats over the rounds: batches {d['batches']}, "
              f"[1] pipelined {d['speculative_submits']}, [2] redone {d['speculative_redone']}")
    print(f"  gen - plain: {med['gen'] - med['plain']:+.3f} ms/batch ({(med['gen'] / med['plain'] - 1) * 100:+.2f} %)")

    # kernel device times, a pass of its own under the profiler
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run("gen", False)
        run("plain", False)
    tot = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA":
            key = "position_kernel" if "position_kernel" in ev.name else "decode_tile_kernel" if "decode_tile_kernel" in ev.name else None
            if key:
                tot.setdefault(key, []).append(ev.time_range.elapsed_us())
    pos = tot.get("position_kernel", [])
    tile = tot.get("decode_tile_kernel", [])
    if pos:
        us = float(np.median(pos))
        print(f"  position_kernel: {len(pos)} launches, median {us:.1f} us per batch; writes {16 * n / 2**20:.1f} MiB of values "
              f"({16 * n / us / 1e3:.0f} GB/s) and reads {4 * n / 2**20:.1f} MiB of record offsets")
    if tile:
        print(f"  decode_tile_kernel: {len(tile)} launches, median {float(np.median(tile)):.1f} us per batch")
    for dec in arms.values():
        dec.close()


if __name__ == "__main__":
    main()
