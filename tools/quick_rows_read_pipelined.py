"""developer tool: the read side of a Spark reader task handing out GPU rows, synchronous against pipelined rows.  1 M
configs[1]-shaped records (oracle.corpus.cfg2_columns: 64 features) are cut at record boundaries into blocks of BLOCK bytes
(64 MiB by default).  The INTEGRATION reader loop: block k is copied into pinned staging slot k % 3 and submitted
(tfr_decode_submit), block k+1 is submitted before block k's rows are read, and every row's offset is touched on the host:
  sync      : submit, then tfr_batch_rows(to_host = 1) when the rows are asked for;
  pipelined : submit, tfr_batch_rows_async(to_host = 1) right behind it, then tfr_batch_rows(to_host = 1).
Each timing is the host clock from the first staged byte to the last block's rows on the host, ending in a synchronise.  The
arms alternate within this one call after a warm-up; a first pass of each copies every row out, and the concatenations must
be identical.  Prints the card name, its power limit and its max SM clock, and the decoder counters [7] / [8] (rows passes
enqueued without a host synchronisation, and of those rebuilt) over the timed passes.  With TFR_TRACE=1 and --trace, one
more pipelined pass runs with profiling on and prints the stage timeline.
usage: quick_rows_read_pipelined.py [N_RECORDS] [BLOCK_BYTES] [REPS] [--trace]"""
import ctypes as C
import os
import subprocess
import sys
import time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from oracle import oracle
from oracle.corpus import cfg2_columns
from spark_tfrecord_b200 import _native

args = [a for a in sys.argv[1:] if not a.startswith("--")]
n = int(args[0]) if len(args) > 0 else 1_000_000
block = int(args[1]) if len(args) > 1 else 64 << 20
reps = int(args[2]) if len(args) > 2 else 5
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))

schema, cols = cfg2_columns(n, seed=4243)
data, rc, _ = oracle.encode(cols, schema)
assert rc == 0
data = np.frombuffer(data, np.uint8)
# block boundaries at record starts (what the carry of the reader loop would give)
starts, pos = [], 0
while pos < len(data):
    starts.append(pos)
    pos += 16 + int(data[pos:pos + 8].view(np.uint64)[0])
cuts, lo = [0], 0
for s in starts:
    if s - lo > block:
        cuts.append(prev)
        lo = prev
    prev = s
cuts.append(len(data))
blocks = [(a, b) for a, b in zip(cuts[:-1], cuts[1:])]
print(f"{n} records, {len(data) / n:.0f} framed bytes each, {len(data) / 2**30:.2f} GiB in {len(blocks)} blocks")

dec = _native.Decoder(schema)
L = _native.lib()
S = _native.Decoder.num_staging_slots()
big = max(b - a for a, b in blocks)
slots = [dec.staging_slot(k, big) for k in range(S)]


def run(pipelined, collect=None):
    rp, op = C.c_void_p(), C.c_void_p()
    nr, nb = C.c_int64(), C.c_size_t()
    touched = 0

    def submit(k):
        a, b = blocks[k]
        st = slots[k % S]
        st[:b - a] = data[a:b]
        h = C.c_void_p()
        _native._check(L.tfr_decode_submit(dec.h, st.ctypes.data, b - a, 0, 1, C.byref(h)))
        if pipelined:
            _native._check(L.tfr_batch_rows_async(h, 1, None, 0, 0, None))
        return h

    ahead = submit(0)
    for k in range(len(blocks)):
        h, ahead = ahead, None
        if k + 1 < len(blocks):
            ahead = submit(k + 1)
        _native._check(L.tfr_batch_rows(h, 1, C.byref(rp), C.byref(op), C.byref(nr), C.byref(nb)))
        offs = np.ctypeslib.as_array(C.cast(op, C.POINTER(C.c_int64)), shape=(nr.value + 1,))
        touched += int(offs.sum() & 1)                         # every row's offset read on the host
        if collect is not None:
            collect.append(C.string_at(rp, nb.value))
            collect.append(offs.tobytes())
        L.tfr_batch_release(h)
    return touched


outs = {}
for name, p in (("sync", False), ("pipelined", True)):
    got = []
    run(p, got)
    outs[name] = b"".join(got)
assert outs["sync"] == outs["pipelined"], "rows differ between the arms"
print(f"rows and offsets: {len(outs['sync']) / 2**30:.3f} GiB, identical for both arms")
for _ in range(2):
    run(False); run(True)
st0 = dec.stats()
times = {"sync": [], "pipelined": []}
for it in range(reps):
    for name, p in (("sync", False), ("pipelined", True)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(p)
        torch.cuda.synchronize()
        times[name].append((time.perf_counter() - t0) * 1e3)
st1 = dec.stats()
print("counters over the timed passes: " + ", ".join(f"{k} {st1[k] - st0[k]}" for k in st1))
for name, ts in times.items():
    print(f"{name:10s}: " + " / ".join(f"{t:.1f}" for t in ts) + f" ms for all {n} records (host clock, staging to host rows, "
          f"ends in a synchronise); median {np.median(ts):.1f} ms, {len(data) / np.median(ts) / 1e6:.1f} GB/s of framed input")
print(f"speed-up of the median: {np.median(times['sync']) / np.median(times['pipelined']):.2f}x")
if "--trace" in sys.argv:
    for name, p in (("sync", False), ("pipelined", True)):
        dec.set_profiling(True)
        run(p)
        print(f"{name} profile (device ms per stage):", dec.get_profile())
        dec.set_profiling(False)
dec.close()
