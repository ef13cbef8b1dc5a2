"""developer tool: tfr_encode_rows on 1 M configs[2] UnsafeRows (about 1.55 KB each), timed on the device with CUDA events
against tfr_encode of the same data as device columns, plus the end-to-end path from pinned row staging to pinned framed
host bytes.  The three are alternated within this one call; the framed outputs must be identical.  Prints the card name
and its power limit.  usage: quick_rows_encode.py [N_ROWS] [REPS]"""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from oracle.corpus import cfg2_columns
from oracle import unsaferow as U
from spark_tfrecord_b200 import _native
from spark_tfrecord_b200._cabi import tfr_column

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))

schema, cols = cfg2_columns(n, seed=4242)
data, offs = U.cfg2_rows(cols)
print(f"{n} rows, {len(data) / n:.0f} bytes of UnsafeRow each, {len(data) / 2**30:.2f} GiB")
# the vectorised rows against the row-by-row builder on the first 10k rows
k = min(n, 10_000)
rows = [tuple(c.get(r) for c in cols) for r in range(k)]
d2, o2 = U.unsafe_rows(schema, rows)
assert np.array_equal(o2, offs[:k + 1]) and np.array_equal(d2, data[:offs[k]]), "cfg2_rows differs from unsafe_rows"

d_rows = torch.from_numpy(data).cuda()
d_offs = torch.from_numpy(offs).cuda()
keep, dcols = [], []
for c in cols:
    t = tfr_column()
    hc = c.to_ctypes()
    for f, _ in tfr_column._fields_:
        setattr(t, f, getattr(hc, f))
    v = torch.from_numpy(c.validity).cuda(); keep.append(v); t.validity = v.data_ptr()
    for l, o in enumerate(c.offsets):
        ot = torch.from_numpy(o).cuda(); keep.append(ot); t.offsets[l] = ot.data_ptr()
    vt = torch.from_numpy(c.values.view(np.uint8)).cuda(); keep.append(vt); t.values = vt.data_ptr()
    dcols.append(t)

enc = _native.Encoder(schema, 0, 0)
stream = torch.cuda.ExternalStream(enc.stream())
staging = enc.row_staging(len(data))
staging[:len(data)] = data
h_offs = offs.copy()


def run_rows():
    enc.encode_rows(d_rows, d_offs)


def run_cols():
    enc.encode_columns(dcols, True)


def run_e2e():
    enc.encode_rows((staging.ctypes.data, len(data), 0), h_offs)
    p, nb = C_result()
    return nb


import ctypes as C
def C_result():
    p = C.c_void_p(); nb = C.c_size_t()
    _native._check(_native.lib().tfr_encoder_result_host(enc.h, C.byref(p), C.byref(nb)))
    return p.value, nb.value


outs = {}
for name, fn in (("rows", run_rows), ("columns", run_cols), ("e2e", run_e2e)):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    outs[name] = enc.result_host()
assert outs["rows"] == outs["columns"] == outs["e2e"], "framed outputs differ"
nb = len(outs["rows"])
print(f"framed output: {nb / 2**30:.3f} GiB, identical for all three paths")

times = {"rows": [], "columns": [], "e2e": []}
for it in range(3):
    for name, fn in (("rows", run_rows), ("columns", run_cols)):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        times[name].append(e0.elapsed_time(e1) / reps)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        run_e2e()
    times["e2e"].append((time.perf_counter() - t0) * 1e3 / reps)
for name, ts in times.items():
    what = "host clock, ends in a synchronise" if name == "e2e" else "CUDA events"
    print(f"{name:8s}: " + " / ".join(f"{t:.3f}" for t in ts) + f" ms per call ({what}); best {len(data) / min(ts) / 1e6:.1f} GB/s of rows, "
          f"{nb / min(ts) / 1e6:.1f} GB/s of framed output")
enc.close()
