"""Large-record decode throughput on one GPU: the image-style, embedding and mixed-outlier corpora of
tests/test_gpu_large_records.py, resident (device input) and end to end (host input, host copy of the columns), GB/s of framed
input, median of --reps alternated runs.  `--arm` selects the path: `large` (this build) or `general` (TFR_DISABLE_FAST: the
path such batches took before the large-record kernel).  Run both arms in one call: python quick_large_records.py --both.
Prints one JSON line per (corpus, arm) with the card's name, SM clock and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))


def corpora():
    from test_gpu_large_records import embed_corpus, image_corpus
    from spark_tfrecord_b200.sqltypes import FloatType
    sch, img = image_corpus(2000, 100_000, seed=1, jitter=40_000)
    sch2, emb = embed_corpus(20_000, 2048, seed=2, elem=FloatType())
    sch3, mix = image_corpus(100_000, 1200, seed=3, jitter=300, outliers=set(range(17, 100_000, 997)))
    return {"image_100KB": (sch, img), "embedding_2048f": (sch2, emb), "mixed_outliers": (sch3, mix)}


def run(arm, reps):
    import torch
    from spark_tfrecord_b200 import _native
    out = {}
    for name, (sch, data) in corpora().items():
        dev = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        res = {}
        for mode in ("resident", "end_to_end"):
            dec = _native.Decoder(sch)
            src = dev if mode == "resident" else data
            for _ in range(3):                                   # learning + warm-up
                b = dec.submit(src); b.wait(); b.release()
            ts = []
            for _ in range(reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                b = dec.submit(src)
                if mode == "end_to_end":
                    b.to_host()
                b.wait()
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
                b.release()
            st = dec.stats()
            dec.close()
            ts.sort()
            res[mode] = round(len(data) / ts[len(ts) // 2] / 1e9, 2)
            res[mode + "_stats"] = {k: st[k] for k in ("speculative_submits", "general_path_batches", "large_record_batches")}
        out[name] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", default="large")
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--both", action="store_true")
    a = ap.parse_args()
    if not a.both:
        print(json.dumps(run(a.arm, a.reps)))
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": q}))
    for r in range(a.rounds):                                    # both arms alternated, each in a fresh process
        for arm in ("general", "large"):
            env = dict(os.environ)
            if arm == "general":
                env["TFR_DISABLE_FAST"] = "1"
            else:
                env.pop("TFR_DISABLE_FAST", None)
            p = subprocess.run([sys.executable, __file__, "--arm", arm, "--reps", str(a.reps)], env=env, capture_output=True, text=True)
            print(json.dumps({"round": r, "arm": arm, "result": json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else p.stderr[-2000:]}))


if __name__ == "__main__":
    main()
