"""Time the mapper's ISAM2 step on the host optimiser (IncrementalOptimizer on SfmWindowProblem) against the device one
(DeviceIncrementalOptimizer, dfk_window_problem_isam2_update / dfk_window_map_steps).

Windows of K keyframes of one synthetic 160x120 scene (two levels, C = 32), LASTN 4 (every keyframe's pairs to its
four predecessors, both ways), perturbed poses, threshold 0.05f as the reference's mapper uses it.  Per scenario and
optimiser: the wall clock of one update (median of the updates after the first, full one), the device time inside it
(torch.profiler, CUDA kernels summed), the kernel launches (the library's launch counter) and the host
synchronisations the profiler sees (stream / device syncs and blocking copies, less the measurement's own).
Scenarios: K = 20 / 50 / 200;
an appended keyframe (grow_problem, then one update); a loop closure (pairs (K, 0) and (0, K) to the new keyframe) added the same way; and a
map_steps run over pho_iters = {15, 15, 15, 30} (device) against mapping_steps (host).

    python tools/bench_mapping.py [--ks 20,50,200] [--updates 6]

Prints one table; run it on the GPU whose numbers you report and note its name and power limit beside them."""
import argparse
import ctypes as C
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deepfactors_b200 import _lib, se3, synth  # noqa: E402
from deepfactors_b200.aligners import SfmAligner  # noqa: E402
from deepfactors_b200.window_opt import (DeviceIncrementalOptimizer, IncrementalOptimizer, OptimizeWork,  # noqa: E402
                                         SfmWindowProblem, mapping_steps)

CS, LEVELS, THRESHOLD = 32, 2, float(np.float32(0.05))


def lastn(K, n=4):
    return [p for k in range(1, K) for m in range(max(0, k - n), k) for p in ((k, m), (m, k))]


class Scene:
    def __init__(self, torch, K):
        base = synth.make_pair(160, 120, CS, LEVELS, seed=5)
        self.cams = [L.cam for L in base.levels]
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
        shared = [dict(img=up(L.img0), grad=up(synth.sobel_np(L.img0)), prx_orig=up(L.prx_orig),
                       prx_jac=up(L.prx_jac)) for L in base.levels]
        self.kf = [[dict(lv, dpt=torch.zeros_like(lv["img"]), valid=torch.zeros_like(lv["img"])) for lv in shared]
                   for _ in range(K)]
        rng = np.random.default_rng(K)
        self.poses = np.stack([se3.identity(np.float64)] + [se3.make_pose(rng.standard_normal(3) * 0.003,
                                                                          rng.standard_normal(3) * 0.01, np.float64)
                                                            for _ in range(K - 1)])
        self.codes = np.zeros((K, CS))
        self.al = SfmAligner(CS)

    def problem(self, K, extra=()):
        return SfmWindowProblem(self.al, self.cams, self.kf[:K], lastn(K) + list(extra))


def timed(torch, fn):
    """(result, wall ms, device ms, host synchronisations) of fn(): the synchronisations are the stream / device syncs
    and the blocking device-to-host copies the profiler sees"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
    ev = prof.events()
    dev = sum(e.device_time_total for e in ev if e.device_type.name == "CUDA" and "Memcpy" not in e.name) / 1e3
    syncs = sum(1 for e in ev if e.name in ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaMemcpy")) - 1
    return out, wall, dev, syncs


def launches(al):
    ms, main, total = C.c_double(), C.c_uint64(), C.c_uint64()
    _lib.lib().dfk_get_profile(al.handle, C.byref(ms), C.byref(main), C.byref(total))
    return int(total.value)


def run(torch, K, updates):
    rows = []
    sc = Scene(torch, K + 1)
    for name in ("host", "device"):
        prob = sc.problem(K)
        if name == "host":
            opt = IncrementalOptimizer.from_problem(prob, sc.poses[:K], sc.codes[:K], relinearize_threshold=THRESHOLD)
        else:
            opt = DeviceIncrementalOptimizer(prob, relinearize_threshold=THRESHOLD, poses=sc.poses[:K],
                                             codes=sc.codes[:K])
        launches(sc.al)
        res = []
        for _ in range(updates):
            r, wall, dev, syncs = timed(torch, opt.update)
            res.append((wall, dev, launches(sc.al), syncs, r))
        steady = res[1:]
        rows.append((f"K={K} update", name, statistics.median(w for w, *_ in steady),
                     statistics.median(d for _, d, *_ in steady), statistics.median(n for _, _, n, *_ in steady),
                     statistics.median(s for *_, s, _ in steady), res[-1][4].factors_relinearised))
        # an appended keyframe and a loop closure: grow, then one update
        for what, extra in (("append", ()), ("loop", ((K, 0), (0, K)))):
            new = sc.problem(K + 1, extra)
            old_pairs = {p: i for i, p in enumerate(prob.pairs)}
            factor_of = [old_pairs.get(p) for p in new.pairs]
            grow = lambda: opt.grow_problem(prob, new, sc.poses[:K + 1], sc.codes[:K + 1], None, factor_of, [])
            _, gwall, gdev, gs = timed(torch, grow)
            launches(sc.al)
            r, wall, dev, syncs = timed(torch, opt.update)
            rows.append((f"K={K} {what} + update", name, gwall + wall, gdev + dev, launches(sc.al), gs + syncs,
                         r.factors_relinearised))
            prob = new
    # map_steps over pho_iters = {15, 15, 15, 30}: the schedule has LEVELS levels, so its last LEVELS entries
    iters = [15, 15, 15, 30][-LEVELS:]
    for name in ("host", "device"):
        prob = sc.problem(K)
        works = [OptimizeWork(iters) for _ in prob.dense_pairs()]
        if name == "host":
            opt = IncrementalOptimizer.from_problem(prob, sc.poses[:K], sc.codes[:K], relinearize_threshold=THRESHOLD)
            fn = lambda: mapping_steps(opt, prob, works, 200)
        else:
            opt = DeviceIncrementalOptimizer(prob, relinearize_threshold=THRESHOLD, poses=sc.poses[:K],
                                             codes=sc.codes[:K])
            fn = lambda: opt.map_steps(works, 200)
        launches(sc.al)
        (res, _), wall, dev, syncs = timed(torch, fn)
        n = max(len(res), 1)
        rows.append((f"K={K} map_steps ({len(res)} steps), per step", name, wall / n, dev / n, launches(sc.al) / n,
                     syncs / n, sum(r.factors_relinearised for r in res) / n))
    return rows


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="20,50,200")
    ap.add_argument("--updates", type=int, default=6)
    a = ap.parse_args()
    print(f"GPU: {torch.cuda.get_device_name()}; C = {CS}, {LEVELS} levels, 160x120, LASTN 4")
    print(f"{'scenario':40s} {'optimiser':9s} {'wall ms':>9s} {'device ms':>10s} {'launches':>9s} {'syncs':>6s} "
          f"{'factors':>8s}")
    for K in (int(k) for k in a.ks.split(",")):
        for r in run(torch, K, a.updates):
            print(f"{r[0]:40s} {r[1]:9s} {r[2]:9.2f} {r[3]:10.2f} {r[4]:9.0f} {r[5]:6.1f} {r[6]:8.1f}")


if __name__ == "__main__":
    main()
