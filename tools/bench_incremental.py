"""Incremental window solve (dfk_window_solver_update) against a full refactorisation, per update: wall clock (the call
synchronises once, so a host clock around it plus a device synchronise covers the work), summed device time (a separate
torch.profiler run) and kernel launches.

Windows of K = 20, 50, 200 keyframes at C = 32 with LASTN 4 back connections (both directions) and one loop link
(K - 1, 2), random positive definite records.  Each case alternates two buffers that differ only in the terms of the
keyframes a mapping step changes, so every timed update re-factorises from the same column:
  full       keyframe 0 changes: j0 = 0, every column (a fresh solver's work, plus the compare and the read-back)
  append     the last 4 keyframes change (a new keyframe's back connections): j0 = K - 4
  loop       keyframe 2 changes (the loop link's lower end): j0 = 2
and `solve` is dfk_window_solve of the same window at lambda = 0 for scale.  One JSON line per (K, case), with the card's
name and power limit, and the device time per update split by kernel (load, compare, replay, panel, update, finish,
backward, ...) from the same profiled run.

    python tools/bench_incremental.py [--reps 50] [--sizes 20 50 200] [--code-size 32]
"""
import argparse
import ctypes as C
import json
import os
import re
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def lastn_pairs(K, n=4):
    return [p for k in range(1, K) for m in range(max(0, k - n), k) for p in ((k, m), (m, k))]


def window_case(al, K, cs, rng):
    from deepfactors_b200.aligners import Window
    from deepfactors_b200.factors import WindowBlocks
    pairs = lastn_pairs(K) + [(0, 0)]
    links = [(K - 1, 2)]
    layout = WindowBlocks(K, cs, pairs, links)
    NP, NG = 12 + cs, 12 + 2 * cs
    A = rng.standard_normal((len(pairs), 2 * NP, NP + 1))
    G = rng.standard_normal((1, 2 * NG, NG + 1))
    recs = (np.einsum("nri,nrj->nij", A[..., :NP], A[..., :NP]).astype(np.float32),
            np.einsum("nri,nr->ni", A[..., :NP], A[..., NP]).astype(np.float32),
            np.ones(len(pairs), np.float32), np.full(len(pairs), 100))
    geo = (np.einsum("nri,nrj->nij", G[..., :NG], G[..., :NG]).astype(np.float32),
           np.einsum("nri,nr->ni", G[..., :NG], G[..., NG]).astype(np.float32), np.ones(1, np.float32))
    buf = layout.pack(list(range(len(pairs))), *recs, [(4, 4)] * len(pairs), geo=geo)
    win = Window(al, K, pairs, list(range(len(pairs))), [(4, 4)] * len(pairs), links)
    return layout, win, buf


def touched(layout, buf, kfs, rng):
    out = buf.copy()
    B = layout.B
    D = out[:layout.num_keyframes * B * B].reshape(-1, B, B)
    for j in kfs:
        A = rng.standard_normal((B, B)).astype(np.float32) * 0.1
        D[j] += A @ A.T
    return out


def power_limit_w():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--sizes", type=int, nargs="+", default=[20, 50, 200])
    ap.add_argument("--code-size", type=int, default=32)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    from deepfactors_b200.window_opt import diag_eps_of
    if not torch.cuda.is_available():
        raise SystemExit("bench_incremental needs a CUDA device")
    card = {"gpu": torch.cuda.get_device_properties(0).name, "power_limit_w": power_limit_w()}
    cs = args.code_size
    al = SfmAligner(cs)
    L = _lib.lib()

    def launches():
        ms, n1, total = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
        _lib.check(al.handle, L.dfk_get_profile(al.handle, C.byref(ms), C.byref(n1), C.byref(total)))
        return int(total.value)

    for K in args.sizes:
        rng = np.random.default_rng(K)
        layout, win, base = window_case(al, K, cs, rng)
        fixed = tuple(range(6))
        eps = diag_eps_of(layout, base, fixed)
        sol = WindowSolver(win, fixed)
        cases = {"full": [0], "append": list(range(K - 4, K)), "loop": [2]}
        for name, kfs in list(cases.items()) + [("solve", None)]:
            if kfs is None:
                b = torch.from_numpy(base).cuda()

                def call():
                    sol.solve(b, 0.0)
                first = 0
            else:
                bufs = [torch.from_numpy(base).cuda(), torch.from_numpy(touched(layout, base, kfs, rng)).cuda()]
                state = {"i": 0}

                def call():
                    state["i"] ^= 1
                    return sol.update(bufs[state["i"]], eps)[1]
                sol.update(bufs[0], eps)
                first = call()
            for _ in range(3):  # warm-up
                call()
            torch.cuda.synchronize()
            launches()
            call()
            torch.cuda.synchronize()
            per_call = launches()
            t0 = time.perf_counter()
            for _ in range(args.reps):
                call()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) / args.reps * 1e6
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    call()
                torch.cuda.synchronize()
            dev = sum(e.self_device_time_total for e in prof.key_averages()) / args.reps
            split = {}  # device time per update of each kernel (copies and memsets under their own names)
            for e in prof.key_averages():
                m = re.search(r"(window_\w+?_kernel)", e.key)
                k = m.group(1) if m else e.key[:40]
                split[k] = split.get(k, 0.0) + e.self_device_time_total / args.reps
            split = {k: round(v, 1) for k, v in sorted(split.items(), key=lambda kv: -kv[1]) if v >= 0.05}
            print(json.dumps({"bench": "window_incremental", "K": K, "C": cs, "tiles": sol.tiles, "case": name,
                              "first_column": first, "wall_us": round(wall, 1), "device_us": round(dev, 1),
                              "launches": per_call, "device_us_by_kernel": split, **card}), flush=True)


if __name__ == "__main__":
    main()
