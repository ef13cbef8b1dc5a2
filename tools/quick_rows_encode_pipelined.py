"""developer tool: the row-to-bytes leg of a Spark writer task, synchronous against pipelined.  1 M configs[2] UnsafeRows
(about 1.55 KB each) are cut into flushes of FLUSH rows (64 Ki by default).  Per flush, the rows are staged into pinned
row staging (the copy the JVM's write(row) does) and encoded to pinned framed host bytes:
  sync      : staging slot 0, tfr_encode_rows + tfr_encoder_result_host, one flush after the other;
  pipelined : staging slot k % S, tfr_encode_rows_submit, and tfr_encoded_wait on the flush that used slot k before it is
              refilled (the RowWriter loop of INTEGRATION.md), so all S slots are in flight.
Each timing is the host clock from the first staged byte to the last framed host byte, ending in a synchronise.  The two arms
alternate within this one call after a warm-up; a first pass of each copies every flush's bytes out, and the concatenations
must be identical.  Prints the card name, its power limit and its max SM clock.
usage: quick_rows_encode_pipelined.py [N_ROWS] [FLUSH_ROWS] [REPS]"""
import ctypes as C
import os
import subprocess
import sys
import time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from oracle.corpus import cfg2_columns
from oracle import unsaferow as U
from spark_tfrecord_b200 import _native

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
flush = int(sys.argv[2]) if len(sys.argv) > 2 else 65_536
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))

schema, cols = cfg2_columns(n, seed=4242)
data, offs = U.cfg2_rows(cols)
cuts = list(range(0, n, flush)) + [n]
flushes = []
for a, b in zip(cuts[:-1], cuts[1:]):
    lo, hi = int(offs[a]), int(offs[b])
    flushes.append((lo, hi, (offs[a:b + 1] - offs[a]).astype(np.int32)))
print(f"{n} rows, {len(data) / n:.0f} bytes of UnsafeRow each, {len(data) / 2**30:.2f} GiB in {len(flushes)} flushes of {flush} rows")

enc = _native.Encoder(schema, 0, 0)
L = _native.lib()
S = _native.Encoder.num_row_slots()
big = max(hi - lo for lo, hi, _ in flushes)
slots = [enc.row_staging_slot(k, big) for k in range(S)]


def run_sync(collect=None):
    out_p, nb = C.c_void_p(), C.c_size_t()
    er = C.c_int64()
    for lo, hi, o in flushes:
        st = slots[0]
        st[:hi - lo] = data[lo:hi]
        _native._check(L.tfr_encode_rows(enc.h, st.ctypes.data, o.ctypes.data, len(o) - 1, 0, C.byref(out_p), C.byref(nb), C.byref(er)))
        _native._check(L.tfr_encoder_result_host(enc.h, C.byref(out_p), C.byref(nb)))
        if collect is not None:
            collect.append(C.string_at(out_p, nb.value))


def run_pipelined(collect=None):
    pending = [None] * S
    p, nb = C.c_void_p(), C.c_size_t()
    er = C.c_int64()

    def drain(k):
        h = pending[k]
        _native._check(L.tfr_encoded_wait(h, C.byref(er)))
        _native._check(L.tfr_encoded_result(h, 1, C.byref(p), C.byref(nb)))
        if collect is not None:
            collect.append(C.string_at(p, nb.value))
        L.tfr_encoded_release(h)
        pending[k] = None

    for i, (lo, hi, o) in enumerate(flushes):
        k = i % S
        if pending[k] is not None:
            drain(k)
        st = slots[k]
        st[:hi - lo] = data[lo:hi]
        h = C.c_void_p()
        _native._check(L.tfr_encode_rows_submit(enc.h, st.ctypes.data, o.ctypes.data, len(o) - 1, 0, C.byref(h)))
        pending[k] = h
    for j in range(len(flushes), len(flushes) + S):
        if pending[j % S] is not None:
            drain(j % S)


outs = {}
for name, fn in (("sync", run_sync), ("pipelined", run_pipelined)):
    got = []
    fn(got)
    outs[name] = b"".join(got)
assert outs["sync"] == outs["pipelined"], "framed outputs differ"
nb_out = len(outs["sync"])
print(f"framed output: {nb_out / 2**30:.3f} GiB, identical for both arms")
for _ in range(2):
    run_sync(); run_pipelined()
st0 = enc.stats()
times = {"sync": [], "pipelined": []}
for it in range(reps):
    for name, fn in (("sync", run_sync), ("pipelined", run_pipelined)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times[name].append((time.perf_counter() - t0) * 1e3)
st1 = enc.stats()
print("pipelined stats over the timed passes: " + ", ".join(f"{k} {st1[k] - st0[k]}" for k in st1))
for name, ts in times.items():
    print(f"{name:10s}: " + " / ".join(f"{t:.1f}" for t in ts) + f" ms for all {n} rows (host clock, staging to framed host bytes, "
          f"ends in a synchronise); median {np.median(ts):.1f} ms, {len(data) / np.median(ts) / 1e6:.1f} GB/s of rows")
print(f"speed-up of the median: {np.median(times['sync']) / np.median(times['pipelined']):.2f}x")
enc.close()
