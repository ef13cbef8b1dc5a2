"""Times the rows pass (profile stage 7: size kernel, scan, emit kernel) with and without partition values, in one process,
arms alternated round by round:
  (p) another build of the library (--parent-lib, e.g. the parent commit's), tfr_batch_rows
  (0) this library, tfr_batch_rows (np = 0)
  (w) this library, tfr_batch_rows_with_partition with a 10-byte date string and an int partition column
Workload: 1 M configs[1]/[2] records (oracle.corpus.cfg2_columns), decoded from device memory.  The rows of (p) and (0) must
be identical, and those of (w) equal to tests/partition_rows.cfg2_joined_rows.  Prints the card, its power limit and max SM
clock, and per arm the median, min and max of the rounds.

usage: python tools/quick_rows_partition.py [--parent-lib PATH] [N_ROWS] [ROUNDS]
(for the parent commit: build its libtfrgpu.so into a directory outside the package and put its _native.py beside it)"""
import importlib.util
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
import partition_rows as P  # noqa: E402

PART = (["string", "int"], ["2024-05-01", 20240501])


class _Dev:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def native_from(lib_path):
    """a second copy of the binding, bound to another build of the library: the _native.py beside that library (the
    binding of the same commit, which declares no symbol the library lacks), else this one"""
    src = os.path.join(os.path.dirname(os.path.abspath(lib_path)), "_native.py")
    old = os.environ.get("TFR_LIB")
    os.environ["TFR_LIB"] = lib_path
    try:
        spec = importlib.util.spec_from_file_location("spark_tfrecord_b200._native_other", src if os.path.exists(src) else _native.__file__)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if old is None:
            del os.environ["TFR_LIB"]
        else:
            os.environ["TFR_LIB"] = old
    mod.lib()
    return mod


def rows_pass(dec, dev, n_bytes, part):
    """one decode + rows; -> (stage-7 ms, (rows, offsets) on the host)"""
    dec.set_profiling(True)
    b, _ = dec.decode((dev.data_ptr(), n_bytes, 1))
    rp, op, n, nb = b.unsafe_rows(False) if part is None else b.unsafe_rows(False, part)
    ms = dec.get_profile()["ms"]["rows"]
    dec.set_profiling(False)
    offs = torch.as_tensor(_Dev(op, n + 1, "<i8"), device="cuda").cpu().numpy().copy()
    rows = torch.as_tensor(_Dev(rp, nb, "|u1"), device="cuda").cpu().numpy().copy()
    b.release()
    return ms, (rows, offs)


def main():
    args = sys.argv[1:]
    parent = None
    if "--parent-lib" in args:
        i = args.index("--parent-lib")
        parent = args[i + 1]
        del args[i:i + 2]
    n = int(args[0]) if args else 1_000_000
    rounds = int(args[1]) if len(args) > 1 else 3
    print(f"card: {card()}  (name, power limit, max SM clock); {rounds} alternated rounds after one warm-up")
    sch, cols = corpus.cfg2_columns(n, seed=1)
    data, rc, _ = oracle.encode(cols, sch)
    assert rc == 0
    want_w = P.cfg2_joined_rows(cols, *PART)
    del cols
    dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    part = (P.partition_row(*PART), P.var_flags(PART[0]))
    arms = {"0": (_native.Decoder(sch), None)}
    if parent:
        arms["p"] = (native_from(parent).Decoder(sch), None)
    arms["w"] = (_native.Decoder(sch), part)
    t = {k: [] for k in arms}
    out = {}
    for rep in range(rounds + 1):                            # round 0 warms every arm up
        for k, (dec, pa) in arms.items():
            ms, rows = rows_pass(dec, dev, len(data), pa)
            if rep:
                t[k].append(ms)
            else:
                out[k] = rows
    for dec, _ in arms.values():
        dec.close()
    ok = np.array_equal(out["w"][0], want_w[0]) and np.array_equal(out["w"][1], want_w[1])
    if parent:
        ok = ok and np.array_equal(out["p"][0], out["0"][0]) and np.array_equal(out["p"][1], out["0"][1])
    names = {"p": "parent library, tfr_batch_rows", "0": "this library, tfr_batch_rows",
             "w": "this library, + partition (string, int)"}
    row_b = {k: int(v[1][1]) for k, v in out.items()}
    for k in arms:
        v = np.array(t[k])
        print(f"  ({k}) {names[k]:42s} rows pass {np.median(v):.3f} ms (min {v.min():.3f}, max {v.max():.3f}), {row_b[k]} B/row")
    base = np.median(t["0"])
    print(f"  with partition / without: time x{np.median(t['w']) / base:.4f}, bytes x{row_b['w'] / row_b['0']:.4f}")
    print(f"  rows equal (parent == this, np = 0; partition rows == cfg2_joined_rows): {ok}")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
