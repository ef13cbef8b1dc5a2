"""Times tfr_batch_rows (a decoded batch as Spark UnsafeRows) next to the Arrow paths, in one process, arms alternated:
  (a) tfr_decode of device-resident framed bytes to device columns
  (b) the same followed by tfr_batch_rows(to_host=0); the rows pass alone is profile stage 7
  (c) pinned staging -> tfr_decode -> tfr_batch_to_host
  (d) pinned staging -> tfr_decode -> tfr_batch_rows(to_host=1)
Workloads: configs[1]/[2] records (oracle.corpus.cfg2_columns), configs[3] SequenceExamples (cfg4_columns), ByteArray
records of 1 KiB.  The rows of (b) and (d) must be identical, and for configs[1]/[2] equal to unsaferow.cfg2_rows of the
source columns.  Prints the card, its power limit and max SM clock with the numbers.

usage: python tools/quick_rows_decode.py [N_ROWS] [REPS]"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import corpus, oracle, unsaferow as U  # noqa: E402
from spark_tfrecord_b200 import _cabi as A, _native  # noqa: E402
from spark_tfrecord_b200.sqltypes import TFR_RT_BYTE_ARRAY, TFR_RT_SEQUENCE_EXAMPLE, TFR_T_BINARY, byte_array_schema  # noqa: E402

HBM_TBS = 3.35            # H100 SXM data sheet, HBM3


class _Dev:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def workloads(n):
    sch, cols = corpus.cfg2_columns(n, seed=1)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0
    wr, wo = U.cfg2_rows(cols)
    yield "configs[1]/[2]", sch, 0, data, (wr, wo.astype(np.int64))
    del cols, wr, wo
    m = max(n // 8, 1)
    sch, cols = corpus.cfg4_columns(m, seed=2)
    data, rc, _ = oracle.encode(cols, sch, TFR_RT_SEQUENCE_EXAMPLE)
    assert rc == 0
    yield "configs[3] SequenceExample", sch, TFR_RT_SEQUENCE_EXAMPLE, data, None
    m = max(n // 2, 1)
    rng = np.random.default_rng(3)
    payload = rng.integers(0, 256, (m, 1024), dtype=np.uint8)
    # framed with the oracle's writer (the ByteArray decoder verifies the payload CRCs)
    sch = byte_array_schema()
    cols = [A.HostColumn(TFR_T_BINARY, 0, m, np.full((m + 7) // 8, 0xFF, np.uint8), [np.arange(m + 1, dtype=np.int32) * 1024], payload.reshape(-1))]
    data, rc, _ = oracle.encode(cols, sch, TFR_RT_BYTE_ARRAY)
    assert rc == 0
    yield "ByteArray 1 KiB", sch, TFR_RT_BYTE_ARRAY, data, None


def run(name, sch, rt, data, want, reps):
    dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    dec = _native.Decoder(sch, rt)
    stage = dec.staging(len(data))
    stage[:len(data)] = np.frombuffer(data, np.uint8)
    t = {k: [] for k in "abcd"}
    rows_ms, info = [], None
    b_rows = d_rows = None
    for rep in range(reps + 1):                                # rep 0 warms every arm up
        torch.cuda.synchronize()
        t0 = time.perf_counter(); b, _ = dec.decode((dev.data_ptr(), len(data), 1)); dt = time.perf_counter() - t0
        info = b.info; b.release(); t["a"].append(dt)
        dec.set_profiling(True)
        t0 = time.perf_counter(); b, _ = dec.decode((dev.data_ptr(), len(data), 1)); rp, op, n, nb = b.unsafe_rows(False)
        dt = time.perf_counter() - t0
        rows_ms.append(dec.get_profile()["ms"]["rows"]); dec.set_profiling(False); t["b"].append(dt)
        if rep == 0:
            offs = torch.as_tensor(_Dev(op, n + 1, "<i8"), device="cuda").cpu().numpy().copy()
            rows = torch.as_tensor(_Dev(rp, nb, "|u1"), device="cuda").cpu().numpy().copy() if nb else np.zeros(0, np.uint8)
            b_rows = (rows, offs)
        b.release()
        t0 = time.perf_counter(); b, _ = dec.decode(stage, nbytes=len(data)); b.to_host_raw(); dt = time.perf_counter() - t0
        b.release(); t["c"].append(dt)
        t0 = time.perf_counter(); b, _ = dec.decode(stage, nbytes=len(data)); r, o = b.unsafe_rows(True); dt = time.perf_counter() - t0
        if rep == 0:
            d_rows = (r.copy(), o.copy())
        b.release(); t["d"].append(dt)
    dec.close()
    same = np.array_equal(b_rows[0], d_rows[0]) and np.array_equal(b_rows[1], d_rows[1])
    oracle_ok = None if want is None else (np.array_equal(b_rows[0], want[0]) and np.array_equal(b_rows[1], want[1]))
    n = info["n_rows"]
    nb = int(b_rows[1][-1])
    med = {k: 1e3 * float(np.median(v[1:])) for k, v in t.items()}
    rms = float(np.median(rows_ms[1:]))
    moved = info["out_bytes"] + nb
    gbs = moved / (rms * 1e-3) / 1e9
    print(f"{name}: {n} records, {len(data) / n:.1f} framed B/record, {info['out_bytes'] / n:.1f} Arrow B/record, {nb / n:.1f} row B/record")
    print(f"  (a) device bytes -> tfr_decode                 {med['a']:9.2f} ms")
    print(f"  (b) (a) + tfr_batch_rows(to_host=0)            {med['b']:9.2f} ms   rows pass (stage 7) {rms:.3f} ms")
    print(f"  (c) pinned staging -> tfr_batch_to_host        {med['c']:9.2f} ms")
    print(f"  (d) pinned staging -> tfr_batch_rows(to_host=1){med['d']:9.2f} ms")
    print(f"  rows pass: {moved / 1e9:.3f} GB (Arrow read + rows written) in {rms:.3f} ms = {gbs:.0f} GB/s, "
          f"{100 * gbs / (HBM_TBS * 1e3):.1f} % of the {HBM_TBS} TB/s data-sheet HBM bandwidth (this kernel group's share)")
    print(f"  rows (b) == (d): {same}" + ("" if oracle_ok is None else f"; == unsaferow.cfg2_rows of the source: {oracle_ok}"))
    return same and oracle_ok is not False


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    print(f"card: {card()}  (name, power limit, max SM clock); medians of {reps} alternated rounds")
    ok = True
    for w in workloads(n):
        ok = run(*w, reps) and ok
        torch.cuda.empty_cache()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
