"""Times DBoW2 vocabulary training on the device (aligners.TrainVocabulary, dfk_bow_vocabulary_train) at
voc_builder's configuration (k = 10, L = 6) over synthetic descriptors: a seeded planted hierarchy of centres with
bit-flip noise per level.

    python tools/bench_vocabulary.py [--sizes 250000 2500000] [--bytes 32 48] [--repeats 7] [--oracle-timeout 180]
                                     [--out DIR]

Per workload: the median, least and largest wall time of --repeats calls, each up to a device synchronise (after one
untimed call of the same shape); the most assignment rounds any node of each level made; the summed device time per
kernel from a separate torch.profiler run; the stats of the call; and the sequential C oracle (one host thread) on the
same inputs when it finishes within --oracle-timeout seconds ("not measured" otherwise).  The card's name and power
limit are read in the same run.  Prints one JSON line per workload and writes them to
DIR/bench_vocabulary.json when --out is given."""
import argparse
import json
import multiprocessing as mp
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def _oracle(q, x, off):
    from bow_oracle import bow_oracle as bo
    t = time.perf_counter()
    bo.train(x, off, 10, 6, 0)
    q.put(time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[250000, 2500000])
    ap.add_argument("--bytes", type=int, nargs="+", default=[32, 48])
    ap.add_argument("--oracle-timeout", type=float, default=180.0)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bow_train_cases as bt
    from deepfactors_b200 import aligners as A

    if not torch.cuda.is_available():
        raise SystemExit("bench_vocabulary: no GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    rows = []
    for D in a.bytes:
        for n in a.sizes:
            x = bt.planted(n, D, 10, 5, 6 if D == 32 else 9, seed=n + D)
            off = np.arange(0, n + 1, 1000, dtype=np.int64)
            if off[-1] != n:
                off = np.append(off, n)
            t = torch.from_numpy(x).cuda()
            A.TrainVocabulary(t, 10, 6, 0, image_offsets=off)  # warm-up of the same shape
            torch.cuda.synchronize()
            walls = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                v = A.TrainVocabulary(t, 10, 6, 0, image_offsets=off)
                torch.cuda.synchronize()
                walls.append(time.perf_counter() - t0)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                A.TrainVocabulary(t, 10, 6, 0, image_offsets=off)
                torch.cuda.synchronize()
            kernels = {}
            for e in prof.key_averages():
                m = re.search(r"(\w+_kernel)", e.key)
                if e.device_type.name == "CUDA" and m:
                    name = m.group(1)
                    kernels[name] = kernels.get(name, 0.0) + e.self_device_time_total / 1e3
            q = mp.get_context("fork").Queue()
            p = mp.get_context("fork").Process(target=_oracle, args=(q, x, off))
            p.start()
            p.join(a.oracle_timeout)
            if p.is_alive():
                p.kill()
                p.join()
                oracle = "not measured"
            else:
                oracle = round(q.get(), 3)
            row = dict(card=card, N=n, D=D, k=10, L=6, calls=len(walls), wall_median_s=round(float(np.median(walls)), 4),
                       wall_min_s=round(min(walls), 4), wall_max_s=round(max(walls), 4),
                       rounds_per_level=v.stats["level_max_rounds"][:6],
                       kernel_ms={k: round(v_, 3) for k, v_ in sorted(kernels.items(), key=lambda kv: -kv[1])},
                       stats=v.stats, oracle_one_thread_s=oracle)
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_vocabulary.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
