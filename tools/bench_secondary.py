#!/usr/bin/env python
"""Secondary measurements of SURVEY.md 8(d) -- everything on the path that is NOT bench.py's headline line.

  python tools/bench_secondary.py [--reps 20] > secondary.jsonl

One JSON line per case:
  * SfmAligner::RunStep at the other BASELINE configs: 160x120 C=8 (configs[0]), 640x480 level 0 at C=64 and
    C=128 (config v), batched so that one launch streams more than the 50 MB L2 of an H100; device time by CUDA events.
  * the synchronous per-call API (what a PhotometricFactor / CameraTracker pays per call, including the result
    read-back): SfmAligner::RunStep, EvaluateError, SE3Aligner::RunStep, UpdateDepth, SobelGradients,
    GaussianBlurDown at 640x480 -- wall clock per call.
  * CameraTracker::TrackFrame (19 iterations) and Relocalize against K = 8 / 32 keyframes, per keyframe and batched --
    wall clock per call, and for Relocalize the summed device time.
  * ReprojectionFactor linearisation of K = 32 / 400 factors x 1000 matches at C = 32 / 128: K synchronous
    ReprojectionLinearize calls + the host A^T A (the only route before the batched call) against one
    ReprojectionLinearizeBatch -- wall clock and summed device time; and one linearisation of the window200 window
    (50 keyframes, 200 photometric pairs, 4 levels at 640x480, C = 32) without and with 400 reprojection links.
  * SparseGeometricFactor linearisation of K = 32 / 200 factors x M = 500 / 3000 points at C = 32 / 128, 640x480
    level 0: K synchronous SparseGeometricLinearize calls + the host A^T A against one SparseGeometricLinearizeBatch;
    and one linearisation of the window200 window without and with 50 geometric links x 3000 points.
  * the window solve (`--only solve`): damped_solve(to_dense(buf)) on torch against dfk_window_solve (WindowSolver) on
    random positive definite window buffers of window200 (50 keyframes, 200 pairs of bench.window_pairs) at C = 32 and
    C = 128 and ba2k (200 keyframes, 2000 pairs) at C = 32 -- wall clock to a synchronise, the two alternated; then a
    torch.profiler run of one device solve: device time, launches, and the fp64 flops of the fill pattern over it.
  * tracked frames (`--only frames`): one window200 linearisation + dfk_window_solve (SfmWindowProblem.linearise +
    .solve, 50 keyframes, 200 pairs, 4 levels 640x480, C = 32) without frames and with one frame per keyframe (50
    frames, 200 more RunStep items in the same launch), the device solve alone for both, and one marginalisation of
    the 50 frames (SfmWindowProblem.marginalize: their 200 items re-evaluated + dfk_window_marginalize_frames + the
    read-back): wall clock to a synchronise and summed device time (torch.profiler, separate run).
  * sliding the window (`--only slide`): window200 at C = 32 and 128, one keyframe marginalised
    (dfk_window_marginalize_keyframe alone, and SfmWindowProblem.marginalize_keyframe with the re-evaluation of the
    keyframe's factors), then the device solve of the 49-keyframe slid window with its keyframe prior and without.
  * the window energy without a linearisation (`--only error`): window200 at C = 32 and 128, every keyframe with a
    code-Jacobian pyramid of its own: SfmWindowProblem.error against SfmWindowProblem.linearise with every factor
    stale, dfk_update_depth_batch of the 200 keyframe levels against 200 dfk_update_depth calls, and a 10-iteration LM
    from perturbed poses with the device solve, without and with `error` (its linearisation and error-evaluation
    counts) -- wall clock to a synchronise and summed device time (torch.profiler, separate run); the byte model of
    both paths is printed beside them.
  * the LM loop in the library (`--only lm`): window200 at C = 32 and 128, a 10-iteration LM by DeviceWindowOptimizer
    (dfk_window_lm) against WindowOptimizer(solve=prob.solve) and WindowOptimizer(..., error=prob.error), alternated --
    wall clock to a synchronise and summed device time (torch.profiler, separate run).
  * coarse to fine (`--only levels`): window200's 50 keyframes and 200 pairs at C = 32 and 128 with a 3-level pyramid
    (640x480), a pho_iters = 4,8,15 schedule (dfk_window_lm_levels, 30 steps) against 30 all-level dfk_window_lm steps:
    wall and device time, and from perturbations of increasing size the final pose error and the level-0 energy.
  * keypoint matching of reprojection factors (`--only match`): one keyframe connection (4 back connections x 2
    directions = 8 factors) at 500 ORB-sized and at 1000 BRISK-sized features, and 64 factors at 500: one
    dfk_reprojection_match_batch (wall clock to a synchronise, and summed device time from a separate profiled run)
    against cv2.BFMatcher plus the sequential C RANSAC of match_oracle on the host, factor by factor.
  * ORB features (`--only orb`): 1, 8 and 64 gray images at 256x192 (the network's size) and at 640x480, 500
    features each: one dfk_orb_detect_batch (OrbDetectBatch; wall clock to a synchronise, summed device time and the
    time of each kernel from a separate profiled run) against cv2.ORB_create(500, 1.2, 1).detectAndCompute on the
    host, one image at a time.
  * ORB features with a scale pyramid (`--only orb_pyramid`): 1, 8 and 64 gray images at 640x480, 500 features over 8
    levels of 1.2: one dfk_orb_detect_pyramid_batch (OrbDetectPyramidBatch; wall clock to a synchronise, summed device
    time and the time of each kernel from a separate profiled run) against the sequential C oracle (orb_oracle) and
    cv2.ORB_create(500, 1.2, 8).detectAndCompute on the host, one image at a time.
  * frame preprocessing (`--only preprocess`): 1, 8 and 64 colour frames at 640x480 (the 2x pixel repeat of the two
    test images, each copy with its own noise) to the network's 256x192 with 4 levels and gradients: one
    dfk_preprocess_batch through PreprocessBatch (wall clock to a synchronise, output allocations included) and as a bare
    C call on buffers and items built once (wall clock to a synchronise), summed device time and the time of each kernel
    from a separate profiled run, against cv2.remap + cvtColor + the float conversion on the host (a numpy fp32 product,
    bitwise convertTo; cv2's Python API has no convertTo), one frame at a time with the map computed once.
  * DBoW2 retrieval (`--only bow`): the bag-of-words transform of 1, 8 and 64 frames x 500 random descriptors with the
    reference's small_voc (k 9, L 3, 48 bytes) and an ORB-SLAM-sized vocabulary (k 10, L 6, 32 bytes, random
    centroids, 10^6 words): one dfk_bow_transform_batch (wall clock to a synchronise, and summed device time from a
    separate profiled run) against the sequential C oracle (bow_oracle) on one host thread, frame by frame; and one
    query of a 500-feature frame (max_results 20) against databases of 100, 1,000 and 10,000 entries.  The oracle's
    query scans every entry (no inverted file), so its host time is an upper bound of DBoW2's.
  * keyframe meshes (`--only mesh`): 1, 8 and 64 keyframes at 256x192 and 640x480 with log-stdev, validity and colour
    views and the uint16 depth, from the depth and from the fused decode at C = 32: one dfk_keyframe_mesh_batch as a
    bare C call on buffers and items built once (wall clock to a synchronise), summed device time and the time of each
    kernel from a separate profiled run, the algorithmic bytes and achieved bandwidth over the device time, and the
    sequential C oracle (mesh_oracle) on one host thread from the depth, keyframe by keyframe.
Every line carries the card's name and power limit.  `--only reprojection` / `--only geometric` / `--only solve` /
`--only frames` / `--only slide` / `--only error` / `--only lm` / `--only levels` / `--only match` / `--only orb` /
`--only orb_pyramid` / `--only preprocess` / `--only bow` / `--only mesh` runs those cases alone.
Peak for the roofline fraction: MEASURED_PEAKS.json hbm_gbs (fallback 3350 GB/s, H100 SXM data sheet).
"""
from __future__ import annotations

import argparse
import builtins
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--only", choices=["reprojection", "geometric", "solve", "frames", "slide", "error", "lm", "levels",
                                           "match", "orb", "orb_pyramid", "preprocess", "bow", "mesh"],
                    default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    from deepfactors_b200 import synth
    from deepfactors_b200.aligners import (GaussianBlurDown, SE3Aligner, SfmAligner, SobelGradients, UpdateDepth)

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    ppath = os.path.join(ROOT, "MEASURED_PEAKS.json")
    peak = float(json.load(open(ppath))["hbm_gbs"]) if os.path.exists(ppath) else 3350.0

    props = torch.cuda.get_device_properties(0)
    card = {"gpu": props.name, "power_limit_w": _power_limit_w()}
    _print = builtins.print

    def print(line, **kw):  # noqa: A001 -- every JSON line carries the card it was measured on
        rec = json.loads(line)
        rec.update(card)
        _print(json.dumps(rec), **kw)

    if args.only == "reprojection":
        return reprojection_cases(args, torch, print)
    if args.only == "geometric":
        return geometric_cases(args, torch, print)
    if args.only == "solve":
        return solve_cases(args, torch, print)
    if args.only == "frames":
        return frames_cases(args, torch, print)
    if args.only == "slide":
        return slide_cases(args, torch, print)
    if args.only == "error":
        return error_cases(args, torch, print)
    if args.only == "lm":
        return lm_cases(args, torch, print)
    if args.only == "levels":
        return levels_cases(args, torch, print)
    if args.only == "match":
        return match_cases(args, torch, print)
    if args.only == "orb":
        return orb_cases(args, torch, print)
    if args.only == "orb_pyramid":
        return orb_pyramid_cases(args, torch, print)
    if args.only == "preprocess":
        return preprocess_cases(args, torch, print)
    if args.only == "bow":
        return bow_cases(args, torch, print)
    if args.only == "mesh":
        return mesh_cases(args, torch, print)

    def upload(L):
        d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in dict(
            img0=L.img0, img1=L.img1, dpt0=L.dpt0, prx0_jac=L.prx_jac, grad1=L.grad1, prx_orig=L.prx_orig).items()}
        d["valid0"] = torch.zeros_like(d["img0"])
        d["cam"] = L.cam
        return d

    def batched(w, h, cs, copies, gram="auto"):
        pair = synth.make_pair(w, h, cs, 1, seed=7)
        L = pair.levels[0]
        al = SfmAligner(cs, gram_mode=gram)
        items = []
        keep = []
        for c in range(copies):
            d = upload(L)
            if c:
                d["prx0_jac"] = torch.roll(d["prx0_jac"], shifts=(3 * c, 5 * c), dims=(0, 1)).contiguous()
            keep.append(d)
            items.append(dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, **{k: d[k] for k in (
                "img0", "img1", "dpt0", "valid0", "prx0_jac", "grad1")}))
        work = al.make_work_items(items)
        rec = al.RunStepBatch(work).clone()
        for _ in range(3):
            al.RunStepBatch(work, rec)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            al.RunStepBatch(work, rec)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        bytes_per_launch = copies * w * h * (24 + 4 * cs)
        gbs = bytes_per_launch / (ms * 1e-3) / 1e9
        inl = al.unpack(rec)[0].inliers
        print(json.dumps({"case": f"SfmAligner::RunStep {w}x{h} C={cs} x{copies} items/launch gram={gram}",
                          "ms_per_launch": ms, "evals_per_s": copies / (ms * 1e-3),
                          "algorithmic_MB_per_launch": bytes_per_launch / 1e6, "GBps": gbs, "frac_of_hbm_peak": gbs / peak,
                          "inlier_fraction": inl / (w * h), "timing": "cuda events, includes the finalize kernel"}),
              flush=True)

    batched(160, 120, 8, 256)
    batched(640, 480, 32, 8, "fp32")
    batched(640, 480, 32, 8, "tf32x3")
    batched(640, 480, 64, 4, "fp32")
    batched(640, 480, 64, 4, "tf32x3")
    batched(640, 480, 128, 3, "fp32")
    batched(640, 480, 128, 3, "tf32x3")

    # ---- synchronous per-call API at 640x480 ---------------------------------------------------------------
    pair = synth.make_pair(640, 480, 32, 1, seed=7)
    L = pair.levels[0]
    d = upload(L)
    al = SfmAligner(32)
    se = SE3Aligner()
    code = pair.code
    dpt_out = torch.empty_like(d["dpt0"])
    grad_out = torch.empty_like(d["grad1"])
    half = torch.empty((240, 320), dtype=torch.float32, device=dev)

    def timed(name, fn, bytes_per_call):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.reps * 5):
            fn()
        torch.cuda.synchronize()
        us = (time.perf_counter() - t0) / (args.reps * 5) * 1e6
        print(json.dumps({"case": name + " 640x480 (synchronous call, wall clock)", "us_per_call": us,
                          "algorithmic_MB_per_call": bytes_per_call / 1e6,
                          "GBps": bytes_per_call / (us * 1e-6) / 1e9}), flush=True)

    px = 640 * 480
    timed("SfmAligner::RunStep C=32", lambda: al.RunStep(pair.pose0, pair.pose1, code, L.cam, d["img0"], d["img1"],
                                                         d["dpt0"], None, d["valid0"], d["prx0_jac"], d["grad1"]),
          px * 152)
    timed("SfmAligner::EvaluateError", lambda: al.EvaluateError(pair.pose0, pair.pose1, L.cam, d["img0"], d["img1"],
                                                                d["dpt0"], None, d["grad1"]), px * 12)
    timed("SE3Aligner::RunStep", lambda: se.RunStep(pair.pose1, L.cam, d["img0"], d["img1"], d["dpt0"], d["grad1"]),
          px * 20)
    timed("UpdateDepth C=32", lambda: UpdateDepth(code, d["prx_orig"], d["prx0_jac"], 2.0, dpt_out), px * (8 + 128))
    timed("SobelGradients", lambda: SobelGradients(d["img1"], grad_out), px * 12)
    timed("GaussianBlurDown", lambda: GaussianBlurDown(d["img1"], half), px * 5)

    # ---- CameraTracker::TrackFrame: 3 levels x (10, 5, 4) iterations (data/flags defaults: 19 SE3 steps per frame) --------
    from deepfactors_b200 import se3
    from deepfactors_b200.aligners import CameraTracker, TrackerConfig
    tp = synth.make_pair(640, 480, 8, 3, seed=9)
    lv = [upload(L) for L in tp.levels]
    cams = [L.cam for L in tp.levels]
    iters = (10, 5, 4)
    trk = CameraTracker(cams, TrackerConfig(pyramid_levels=3, iterations_per_level=iters, huber_delta=0.1))
    trk.SetKeyframe([x["img0"] for x in lv], [x["dpt0"] for x in lv])
    img1s, grads = [x["img1"] for x in lv], [x["grad1"] for x in lv]

    def device_loop():
        trk.Reset()
        trk.TrackFrame(img1s, grads)

    def host_loop():  # what the reference does: synchronous step, host solve, next step (camera_tracker.cpp:48-63)
        pose = se3.identity(np.float64)
        for level in (2, 1, 0):
            for _ in range(iters[level]):
                r = se.RunStep(pose.astype(np.float32), cams[level], lv[level]["img0"], lv[level]["img1"], lv[level]["dpt0"],
                               lv[level]["grad1"])
                pose = se3.se3_solve_and_update(r.toDenseMatrix(), r.Jtr, pose)
        return pose

    bytes_track = sum(iters[l] * (640 >> l) * (480 >> l) * 20 for l in range(3))
    timed("CameraTracker::TrackFrame 19 iterations, device-side loop (dfk_se3_track)", device_loop, bytes_track)
    timed("CameraTracker::TrackFrame 19 iterations, per-step API + host solve (reference structure)", host_loop, bytes_track)

    # ---- DeepFactors::Relocalize: the same live frame tracked against K keyframes (deepfactors.cpp:713-743) ---------------
    # K x (SetKeyframe + Reset + TrackFrame), what the reference does, against one Relocalize (dfk_se3_track_batch: one
    # launch per iteration for all K keyframes).  Keyframes: the synthetic keyframe pyramid, every copy rolled by a
    # different offset, each in its own buffers.
    from torch.profiler import ProfilerActivity, profile

    def device_us(fn, reps):  # summed device time (kernels, copies, memsets) per call, from a separate profiled run
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        return sum(e.self_device_time_total for e in prof.key_averages()) / reps

    for K in (8, 32):
        kfs = []
        for k in range(K):
            sh = (7 * k) % 23 - 11
            kfs.append(([torch.roll(x["img0"], shifts=sh >> l, dims=1).contiguous() for l, x in enumerate(lv)],
                        [torch.roll(x["dpt0"], shifts=sh >> l, dims=1).contiguous() for l, x in enumerate(lv)]))

        def per_keyframe():
            errs = []
            for kf in kfs:
                trk.SetKeyframe(kf[0], kf[1])
                trk.Reset()
                trk.TrackFrame(img1s, grads)
                errs.append(trk.GetError())
            return errs

        def relocalize():
            return trk.Relocalize(kfs, img1s, grads)[2]

        assert np.array_equal(np.asarray(per_keyframe(), np.float32), relocalize())  # same errors, bit for bit
        reps = max(2, args.reps // 2)
        for name, fn in (("K x CameraTracker::TrackFrame (dfk_se3_track per keyframe)", per_keyframe),
                         ("one CameraTracker::Relocalize (dfk_se3_track_batch)", relocalize)):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
            us = (time.perf_counter() - t0) / reps * 1e6
            print(json.dumps({"case": f"Relocalize 640x480 live frame vs K={K} keyframes, 3 levels x (10, 5, 4): {name}",
                              "us_per_relocalisation": us, "device_us_per_relocalisation": device_us(fn, reps),
                              "timing": "wall clock (synchronous); device time = summed kernel + copy time, "
                                        "torch.profiler"}), flush=True)

    reprojection_cases(args, torch, print)
    geometric_cases(args, torch, print)


def _power_limit_w():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:  # the number is still worth printing; the limit is then unknown
        return None


def _device_us(torch, fn, reps):
    """summed device time (kernels, copies, memsets) per call, from a separate profiled run"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    return sum(e.self_device_time_total for e in prof.key_averages()) / reps


def _wall_us(torch, fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e6


def reprojection_cases(args, torch, print):
    """ReprojectionFactor linearisation: K x (dfk_reprojection_linearize + host A^T A) against one
    dfk_reprojection_linearize_batch; and a window200 linearisation without / with 400 reprojection links."""
    import numpy as np

    from deepfactors_b200 import se3, synth
    from deepfactors_b200.aligners import ReprojectionLinearize, ReprojectionLinearizeBatch, SfmAligner
    dev = torch.device("cuda", 0)
    M = 1000
    rng = np.random.default_rng(3)

    def matches(cam):  # keypoints of the keyframe and matched keypoints of the frame, ~1 px apart
        q = np.stack([rng.uniform(4, cam.width - 5, M), rng.uniform(4, cam.height - 5, M)], axis=1).astype(np.float32)
        return q, (q + rng.normal(0, 1.0, (M, 2))).astype(np.float32)

    for cs in (32, 128):
        L = synth.make_level(640, 480, cs, seed=12)
        prx = torch.from_numpy(L.prx_orig).to(dev)
        jac = torch.from_numpy(np.ascontiguousarray(L.prx_jac)).to(dev)
        al = SfmAligner(cs)
        for K in (32, 400):
            items = []
            for k in range(K):
                q, t = matches(L.cam)
                items.append(dict(pose0=se3.identity(), pose1=se3.make_pose([0.01 * (k % 5), -0.01, 0.0], [0.05, 0.0, 0.01 * (k % 3)],
                                                                             np.float32),
                                  code0=(rng.standard_normal(cs) * 0.1).astype(np.float32), cam=L.cam, prx_orig=prx,
                                  prx_jac=jac, query_xy=q, train_xy=t, cauchy_delta=1.5, sigma=1.0))
            rec = torch.empty((K, (12 + cs) * (13 + cs) // 2 + 14 + cs), dtype=torch.float32, device=dev)

            def per_factor():  # rows to the host, then A^T A there (what a JacobianFactor costs the solver)
                for it in items:
                    rows, _ = ReprojectionLinearize(al, it["pose0"], it["pose1"], it["code0"], it["cam"], it["prx_orig"],
                                                    it["prx_jac"], it["query_xy"], it["train_xy"], it["cauchy_delta"],
                                                    it["sigma"])
                    r = rows.astype(np.float64)
                    r.T @ r

            def batched():
                ReprojectionLinearizeBatch(al, items, rec)

            for name, fn, reps in ((f"K x ReprojectionLinearize + host A^T A", per_factor, 3 if K > 32 else 5),
                                   (f"one ReprojectionLinearizeBatch", batched, max(5, args.reps))):
                print(json.dumps({"case": f"ReprojectionFactor linearisation C={cs} K={K} factors x {M} matches: {name}",
                                  "us_per_linearisation": _wall_us(torch, fn, reps),
                                  "device_us_per_linearisation": _device_us(torch, fn, reps),
                                  "host_syncs": K if fn is per_factor else 0,
                                  "row_bytes_downloaded": K * 2 * M * (13 + cs) * 4 if fn is per_factor else 0,
                                  "timing": "wall clock (synchronous); device time = summed kernel + copy time, "
                                            "torch.profiler"}), flush=True)

    # ---- window200 (bench.py --config window200): one linearisation of every factor, without and with 400 links --------
    from deepfactors_b200.window_opt import ReprojectionLink, SfmWindowProblem
    sys.path.insert(0, ROOT)
    from bench import window_pairs
    cs, levels, num_kf = 32, 4, 50
    base = synth.make_pair(640, 480, cs, levels, seed=7)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    shared = [dict(img=up(L.img0), grad=up(L.grad1), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac)) for L in base.levels]
    keyframes = [[dict(sh, dpt=torch.zeros_like(sh["img"]), valid=torch.zeros_like(sh["img"])) for sh in shared]
                 for _ in range(num_kf)]
    pairs = window_pairs(num_kf, 200)
    cam0 = base.levels[0].cam
    links = []
    for j in range(400):
        k0, k1 = (int(v) for v in rng.choice(num_kf, 2, replace=False))
        q, t = matches(cam0)
        links.append(ReprojectionLink(k0, k1, q, t, 1.5, 1.0))
    al = SfmAligner(cs)
    poses = np.stack([se3.make_pose([0.001 * (k % 7), 0.0, 0.0], [0.002 * (k % 5), 0.0, 0.0], np.float64)
                      for k in range(num_kf)])
    codes = np.zeros((num_kf, cs))
    for n_links in (0, 400):
        prob = SfmWindowProblem(al, [L.cam for L in base.levels], keyframes, pairs, links=links[:n_links] or None)
        todo = list(range(len(prob.pairs)))

        def lin():
            prob.linearise(poses, codes, todo)

        reps = max(5, args.reps // 2)
        print(json.dumps({"case": f"window200 linearisation (50 keyframes, 200 pairs, 4 levels 640x480, C=32) + {n_links} "
                                  f"reprojection links x {M} matches",
                          "us_per_linearisation": _wall_us(torch, lin, reps),
                          "device_us_per_linearisation": _device_us(torch, lin, reps),
                          "timing": "wall clock to the end of the assembly (synchronised); device time = summed kernel + "
                                    "copy time, torch.profiler"}), flush=True)


def geometric_cases(args, torch, print):
    """SparseGeometricFactor linearisation: K x (dfk_sparse_geometric_linearize + host A^T A) against one
    dfk_sparse_geometric_linearize_batch; and a window200 linearisation without / with 50 geometric links."""
    import numpy as np

    from deepfactors_b200 import _lib, se3, synth
    from deepfactors_b200.aligners import SfmAligner, SparseGeometricLinearize, SparseGeometricLinearizeBatch
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(5)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)

    def points(cam, m):
        return np.stack([rng.integers(2, int(cam.width) - 2, m), rng.integers(2, int(cam.height) - 2, m)], 1).astype(np.int32)

    for cs in (32, 128):
        L0 = synth.make_level(640, 480, cs, seed=21)
        L1 = synth.make_level(640, 480, cs, seed=22, phase=0.3)
        dpt1 = (np.float32(2.0) / L1.prx_orig - np.float32(2.0)).astype(np.float32)
        kf = dict(prx0_orig=up(L0.prx_orig), prx0_jac=up(L0.prx_jac), prx1_orig=up(L1.prx_orig), prx1_jac=up(L1.prx_jac),
                  dpt_grad1=up(synth.sobel_np(dpt1)))
        al = SfmAligner(cs)
        for M in (500, 3000):
            for K in (32, 200):
                items = [dict(pose0=se3.identity(), pose1=se3.make_pose([0.01 * (k % 5), -0.01, 0.0],
                                                                        [0.05, 0.0, 0.01 * (k % 3)], np.float32),
                              code0=(rng.standard_normal(cs) * 0.1).astype(np.float32),
                              code1=(rng.standard_normal(cs) * 0.1).astype(np.float32), cam=L0.cam,
                              points_xy=points(L0.cam, M), huber_delta=0.1, **kf) for k in range(K)]
                rec = torch.empty((K, _lib.geo_record_floats(cs)), dtype=torch.float32, device=dev)

                def per_factor():  # rows to the host, then A^T A there (what a JacobianFactor costs the solver)
                    for it in items:
                        rows, _ = SparseGeometricLinearize(al, it["pose0"], it["pose1"], it["code0"], it["code1"], it["cam"],
                                                           it["prx0_orig"], it["prx0_jac"], it["prx1_orig"], it["prx1_jac"],
                                                           it["dpt_grad1"], it["points_xy"], it["huber_delta"])
                        r = rows.astype(np.float64)
                        r.T @ r

                def batched():
                    SparseGeometricLinearizeBatch(al, items, rec)

                slow = 2 if K * M * cs > 32 * 3000 * 32 else 3
                for name, fn, reps in (("K x SparseGeometricLinearize + host A^T A", per_factor, slow),
                                       ("one SparseGeometricLinearizeBatch", batched, max(5, args.reps))):
                    print(json.dumps({"case": f"SparseGeometricFactor linearisation 640x480 C={cs} K={K} factors x {M} "
                                              f"points: {name}",
                                      "us_per_linearisation": _wall_us(torch, fn, reps),
                                      "device_us_per_linearisation": _device_us(torch, fn, max(1, reps // 2)),
                                      "host_syncs": K if fn is per_factor else 0,
                                      "row_bytes_downloaded": K * M * (13 + 2 * cs) * 4 if fn is per_factor else 0,
                                      "timing": "wall clock (synchronous); device time = summed kernel + copy time, "
                                                "torch.profiler"}), flush=True)
        del kf, items, rec
        torch.cuda.empty_cache()

    # ---- window200 (bench.py --config window200): one linearisation of every factor, without and with 50 links --------
    from deepfactors_b200.window_opt import GeometricLink, SfmWindowProblem
    sys.path.insert(0, ROOT)
    from bench import window_pairs
    cs, levels, num_kf, M = 32, 4, 50, 3000
    base = synth.make_pair(640, 480, cs, levels, seed=7)
    shared = [dict(img=up(L.img0), grad=up(L.grad1), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac)) for L in base.levels]
    dpt = (np.float32(2.0) / base.levels[0].prx_orig - np.float32(2.0)).astype(np.float32)
    shared[0]["dpt_grad"] = up(synth.sobel_np(dpt))  # Sobel of level-0 depth, computed once per keyframe
    keyframes = [[dict(sh, dpt=torch.zeros_like(sh["img"]), valid=torch.zeros_like(sh["img"])) for sh in shared]
                 for _ in range(num_kf)]
    pairs = window_pairs(num_kf, 200)
    cam0 = base.levels[0].cam
    links = []
    for j in range(50):
        k0, k1 = (int(v) for v in rng.choice(num_kf, 2, replace=False))
        links.append(GeometricLink(k0, k1, points(cam0, M), 0.1))
    al = SfmAligner(cs)
    poses = np.stack([se3.make_pose([0.001 * (k % 7), 0.0, 0.0], [0.002 * (k % 5), 0.0, 0.0], np.float64)
                      for k in range(num_kf)])
    codes = np.zeros((num_kf, cs))
    for n_links in (0, 50):
        prob = SfmWindowProblem(al, [L.cam for L in base.levels], keyframes, pairs, geometric=links[:n_links] or None)
        todo = list(range(len(prob.pairs) + n_links))

        def lin():
            prob.linearise(poses, codes, todo)

        reps = max(5, args.reps // 2)
        print(json.dumps({"case": f"window200 linearisation (50 keyframes, 200 pairs, 4 levels 640x480, C=32) + {n_links} "
                                  f"geometric links x {M} points",
                          "us_per_linearisation": _wall_us(torch, lin, reps),
                          "device_us_per_linearisation": _device_us(torch, lin, reps),
                          "timing": "wall clock to the end of the assembly (synchronised); device time = summed kernel + "
                                    "copy time, torch.profiler"}), flush=True)


def frames_cases(args, torch, print):
    """window200 with and without one tracked frame per keyframe: linearisation + device solve, the solve alone, and the
    marginalisation of the 50 frames"""
    import numpy as np
    from deepfactors_b200 import se3, synth
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import SfmWindowProblem, TrackedFrame
    sys.path.insert(0, ROOT)
    from bench import window_pairs
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    cs, levels, num_kf = 32, 4, 50
    base = synth.make_pair(640, 480, cs, levels, seed=7)
    shared = [dict(img=up(L.img0), grad=up(L.grad1), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac)) for L in base.levels]
    keyframes = [[dict(sh, dpt=torch.zeros_like(sh["img"]), valid=torch.zeros_like(sh["img"])) for sh in shared]
                 for _ in range(num_kf)]
    frame_levels = [dict(img=up(L.img1), grad=up(L.grad1)) for L in base.levels]
    frames = [TrackedFrame(k, frame_levels) for k in range(num_kf)]
    pairs = window_pairs(num_kf, 200)
    cams = [L.cam for L in base.levels]
    al = SfmAligner(cs)
    poses = np.stack([se3.make_pose([0.001 * (k % 7), 0.0, 0.0], [0.002 * (k % 5), 0.0, 0.0], np.float64)
                      for k in range(num_kf)])
    fposes = np.stack([se3.make_pose([0.0, 0.001 * (k % 3), 0.0], [0.0, 0.002 * (k % 4), 0.0], np.float64)
                       for k in range(num_kf)])
    codes = np.zeros((num_kf, cs))
    reps = max(5, args.reps // 2)
    fixed = tuple(range(6))
    for n_frames in (0, num_kf):
        prob = SfmWindowProblem(al, cams, keyframes, pairs, frames=frames[:n_frames] or None)
        todo = list(range(len(prob.pairs)))
        fp = fposes[:n_frames] if n_frames else None
        buf, _ = prob.linearise(poses, codes, todo, fp)

        def lin_solve():
            b, _ = prob.linearise(poses, codes, todo, fp)
            prob.solve(b, 1e-4, fixed)

        def solve():
            prob.solve(buf, 1e-4, fixed)

        assert prob.solve(buf, 1e-4, fixed) is not None
        for what, fn in (("linearisation + device solve", lin_solve), ("device solve", solve)):
            print(json.dumps({"case": f"window200 {what} (50 keyframes, 200 pairs, 4 levels 640x480, C=32) + "
                                      f"{n_frames} tracked frames",
                              "us_per_call": _wall_us(torch, fn, reps), "device_us_per_call": _device_us(torch, fn, reps),
                              "timing": "wall clock to a synchronise (the solve reads dx back); device time = summed "
                                        "kernel + copy time, torch.profiler"}), flush=True)
        if n_frames:
            which = list(range(n_frames))

            def marg():
                prob.marginalize(poses, codes, fposes, which)

            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                marg()
                torch.cuda.synchronize()
            kern = sum(e.device_time for e in prof.events()
                       if e.device_type.name == "CUDA" and "window_marginalize" in e.name)
            print(json.dumps({"case": f"window200 marginalisation of {n_frames} tracked frames (their {n_frames * levels} "
                                      "RunStep items re-evaluated + dfk_window_marginalize_frames + read-back)",
                              "us_per_call": _wall_us(torch, marg, reps), "device_us_per_call": _device_us(torch, marg, reps),
                              "marginalize_kernel_us": kern,
                              "timing": "wall clock to a synchronise; device time = summed kernel + copy time, "
                                        "torch.profiler"}), flush=True)


def slide_cases(args, torch, print):
    """window200 at C = 32 and 128: marginalising one keyframe (the device calls alone, and the whole
    SfmWindowProblem.marginalize_keyframe with the re-evaluation of its factors), and the device solve of the 49-keyframe
    window that slides past it, with its keyframe prior and without"""
    import numpy as np
    from deepfactors_b200 import se3, synth
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import SfmWindowProblem, drop_keyframe
    sys.path.insert(0, ROOT)
    from bench import window_pairs
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    levels, num_kf = 4, 50
    reps = max(5, args.reps // 2)
    for cs in (32, 128):
        base = synth.make_pair(640, 480, cs, levels, seed=7)
        shared = [dict(img=up(L.img0), grad=up(L.grad1), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac))
                  for L in base.levels]
        keyframes = [[dict(sh, dpt=torch.zeros_like(sh["img"]), valid=torch.zeros_like(sh["img"])) for sh in shared]
                     for _ in range(num_kf)]
        pairs = window_pairs(num_kf, 200)
        cams = [L.cam for L in base.levels]
        al = SfmAligner(cs)
        poses = np.stack([se3.make_pose([0.001 * (k % 7), 0.0, 0.0], [0.002 * (k % 5), 0.0, 0.0], np.float64)
                          for k in range(num_kf)])
        codes = np.zeros((num_kf, cs))
        prob = SfmWindowProblem(al, cams, keyframes, pairs)
        m = 0
        nb = prob.window.blanket(m)
        prob.linearise(poses, codes, list(range(len(prob.pairs))))
        w = 1e-2

        def dev_only():
            prob.window.marginalize_keyframe(prob.records, m, code_prior_weight=w, code=codes[m])

        def whole():
            prob.marginalize_keyframe(poses, codes, m, code_prior_weight=w)

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            dev_only()
            torch.cuda.synchronize()
        import re
        kern = {}  # kernel -> summed device time of one call
        for e in prof.events():
            k = re.search(r"(window_\w+_kernel)", e.name) if e.device_type.name == "CUDA" else None
            if k:
                kern[k.group(1)] = kern.get(k.group(1), 0.0) + e.device_time
        items = sum(1 for p in pairs if m in p) * levels
        print(json.dumps({"case": f"window200 C={cs}: marginalise keyframe {m} (blanket of {len(nb)}, {items} RunStep "
                                  f"items), dfk_window_marginalize_keyframe alone",
                          "us_per_call": _wall_us(torch, dev_only, reps),
                          "device_us_per_call": _device_us(torch, dev_only, reps), "kernels_us": kern,
                          "timing": "wall clock to a synchronise; device time = summed kernel + copy time, "
                                    "torch.profiler"}), flush=True)
        print(json.dumps({"case": f"window200 C={cs}: SfmWindowProblem.marginalize_keyframe of keyframe {m} (re-evaluation "
                                  "of its factors + the device marginalisation + read-back)",
                          "us_per_call": _wall_us(torch, whole, reps),
                          "device_us_per_call": _device_us(torch, whole, reps),
                          "timing": "wall clock to a synchronise; device time = summed kernel + copy time, "
                                    "torch.profiler"}), flush=True)
        prior = prob.marginalize_keyframe(poses, codes, m, code_prior_weight=w)
        slid = prob.without_keyframe(m, prior)
        bare = SfmWindowProblem(al, cams, keyframes[1:], [p for p in slid.pairs])
        ps, cs_ = drop_keyframe(poses, codes, m)
        fixed = tuple(range(6))
        for name, pr in (("with its keyframe prior", slid), ("without the prior", bare)):
            buf, _ = pr.linearise(ps, cs_, list(range(len(pr.pairs))))
            assert pr.solve(buf, 1e-4, fixed) is not None

            def solve():
                pr.solve(buf, 1e-4, fixed)

            print(json.dumps({"case": f"window200 C={cs}: device solve of the 49-keyframe slid window {name} "
                                      f"({pr._solvers[fixed].tiles} tiles)",
                              "us_per_call": _wall_us(torch, solve, reps),
                              "device_us_per_call": _device_us(torch, solve, reps),
                              "timing": "wall clock to a synchronise (the solve reads dx back); device time = summed "
                                        "kernel + copy time, torch.profiler"}), flush=True)
        del prob, slid, bare, keyframes, shared
        torch.cuda.empty_cache()


def error_cases(args, torch, print):
    """window200 at C = 32 and 128: the window energy by SfmWindowProblem.error against a full linearisation, the batched
    depth decode against one call per keyframe level, and LM without and with `error`"""
    import numpy as np
    from deepfactors_b200 import se3, synth
    from deepfactors_b200.aligners import SfmAligner, UpdateDepth
    from deepfactors_b200.window_opt import LMParams, SfmWindowProblem, WindowOptimizer
    sys.path.insert(0, ROOT)
    from bench import window_pairs
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    levels, num_kf = 4, 50
    reps = max(5, args.reps // 2)
    timing = "wall clock to a synchronise; device time = summed kernel + copy time, torch.profiler (separate run)"
    for cs in (32, 128):
        base = synth.make_pair(640, 480, cs, levels, seed=7)
        shared = [dict(img=up(L.img0), grad=up(L.grad1), prx_orig=up(L.prx_orig)) for L in base.levels]
        jac = [up(L.prx_jac) for L in base.levels]
        gen = torch.Generator(device="cuda").manual_seed(cs)
        # every keyframe its own code Jacobian (the byte model decodes 50 pyramids, not one cached in L2)
        keyframes = [[dict(sh, prx_jac=j + 1e-3 * torch.randn(j.shape, device="cuda", generator=gen),
                           dpt=torch.zeros_like(sh["img"]), valid=torch.zeros_like(sh["img"]))
                      for sh, j in zip(shared, jac)] for _ in range(num_kf)]
        pairs = window_pairs(num_kf, 200)
        cams = [L.cam for L in base.levels]
        al = SfmAligner(cs)
        rng = np.random.default_rng(cs)
        poses = np.stack([se3.make_pose(rng.standard_normal(3) * 0.003, rng.standard_normal(3) * 0.01, np.float64)
                          for _ in range(num_kf)])
        poses[0] = se3.identity(np.float64)
        codes = np.zeros((num_kf, cs))
        prob = SfmWindowProblem(al, cams, keyframes, pairs)
        todo = list(range(len(prob.pairs)))
        px = sum(int(L.img0.size) for L in base.levels)  # pixels of one pyramid
        items = len(pairs) * levels
        bytes_err = num_kf * px * (4 * cs + 8) + len(pairs) * px * 12
        bytes_lin = len(pairs) * px * (4 * cs + 24)
        E, parts = prob.error(poses, codes)
        buf, _ = prob.linearise(poses, codes, todo)
        f = float(buf[prob.layout.offsets()[2]])

        def error():
            prob.error(poses, codes)

        def linearise():
            prob.linearise(poses, codes, todo)
            torch.cuda.synchronize()

        for name, fn, nbytes in (("SfmWindowProblem.error (4 launches + 1 read-back)", error, bytes_err),
                                 ("SfmWindowProblem.linearise, every factor stale", linearise, bytes_lin)):
            wall = _wall_us(torch, fn, reps)
            dev_us = _device_us(torch, fn, reps)
            print(json.dumps({"case": f"window200 C={cs} ({num_kf} keyframes, {len(pairs)} pairs, {levels} levels 640x480, "
                                      f"{items} items): {name}",
                              "us_per_call": wall, "device_us_per_call": dev_us, "bytes_model": nbytes,
                              "model_gbs_over_device_time": nbytes / dev_us / 1e3,
                              "energy": E if fn is error else f, "timing": timing}), flush=True)
        print(json.dumps({"case": f"window200 C={cs}: E against the linearisation's f (valid_border 2: the validity "
                                  "rules differ at the border)", "E": E, "f": f, "parts": parts.__dict__}), flush=True)
        dec = [dict(code=np.zeros(cs, np.float32), prx_orig=kf[l]["prx_orig"], prx_jac=kf[l]["prx_jac"],
                    dpt=kf[l]["dpt"]) for kf in keyframes for l in range(levels)]
        arr = al.make_depth_items(dec)

        def batch():
            al.UpdateDepthBatch(arr)

        def single():
            for it in dec:
                UpdateDepth(it["code"], it["prx_orig"], it["prx_jac"], 2.0, it["dpt"])

        for name, fn in (("one dfk_update_depth_batch", batch), (f"{len(dec)} dfk_update_depth calls", single)):
            print(json.dumps({"case": f"window200 C={cs}: decode {len(dec)} keyframe levels, {name}",
                              "us_per_call": _wall_us(torch, fn, reps), "device_us_per_call": _device_us(torch, fn, reps),
                              "bytes_model": num_kf * px * (4 * cs + 8), "timing": timing}), flush=True)
        prm = LMParams(iterations=10, lambda_init=1e-4)
        for mode in ("linearise", "error"):
            def lm():
                p = SfmWindowProblem(al, cams, keyframes, pairs)
                opt = WindowOptimizer(p.layout, p.linearise, prm, solve=p.solve,
                                      error=p.error if mode == "error" else None)
                return opt.run(poses, codes)

            _, _, tr = lm()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, _, tr = lm()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e6
            dev_us = _device_us(torch, lm, 1)
            print(json.dumps({"case": f"window200 C={cs}: 10-iteration LM from perturbed poses, device solve, "
                                      f"{'with error()' if mode == 'error' else 'linearising every candidate'}",
                              "us_total": wall, "device_us_total": dev_us, "linearisations": tr.linearisations,
                              "error_evaluations": tr.error_evaluations, "accepted": tr.accepted,
                              "energy_first_last": [tr.energy[0], tr.energy[-1]], "timing": timing}), flush=True)
        del prob, keyframes, shared, jac, arr, dec
        torch.cuda.empty_cache()


def lm_cases(args, torch, print):
    """window200 at C = 32 and 128: a 10-iteration LM as one library call (DeviceWindowOptimizer, dfk_window_lm) against
    WindowOptimizer(solve=prob.solve) and WindowOptimizer(..., error=prob.error), alternated, from the same perturbed
    start.  Each optimizer has its own SfmWindowProblem, built (and, for the device loop, device_problem() created) before
    the timed runs: the setup is once per window, the loop once per window update."""
    import numpy as np
    from deepfactors_b200 import se3, synth
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import DeviceWindowOptimizer, LMParams, SfmWindowProblem, WindowOptimizer
    sys.path.insert(0, ROOT)
    from bench import window_pairs
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    levels, num_kf = 4, 50
    reps = max(3, args.reps // 5)
    timing = ("wall clock of one run() to a synchronise, median over the alternated repetitions; device time = summed "
              "kernel + copy time of one run(), torch.profiler (separate run)")
    for cs in (32, 128):
        base = synth.make_pair(640, 480, cs, levels, seed=7)
        shared = [dict(img=up(L.img0), grad=up(L.grad1), prx_orig=up(L.prx_orig)) for L in base.levels]
        jac = [up(L.prx_jac) for L in base.levels]
        gen = torch.Generator(device="cuda").manual_seed(cs)
        keyframes = [[dict(sh, prx_jac=j + 1e-3 * torch.randn(j.shape, device="cuda", generator=gen),
                           dpt=torch.zeros_like(sh["img"]), valid=torch.zeros_like(sh["img"]))
                      for sh, j in zip(shared, jac)] for _ in range(num_kf)]
        pairs = window_pairs(num_kf, 200)
        cams = [L.cam for L in base.levels]
        al = SfmAligner(cs)
        rng = np.random.default_rng(cs)
        poses = np.stack([se3.make_pose(rng.standard_normal(3) * 0.003, rng.standard_normal(3) * 0.01, np.float64)
                          for _ in range(num_kf)])
        poses[0] = se3.identity(np.float64)
        codes = np.zeros((num_kf, cs))
        prm = LMParams(iterations=10, lambda_init=1e-4)
        runs = {}
        for name in ("DeviceWindowOptimizer (dfk_window_lm)", "WindowOptimizer(solve=prob.solve)",
                     "WindowOptimizer(solve=prob.solve, error=prob.error)"):
            p = SfmWindowProblem(al, cams, keyframes, pairs)
            if name.startswith("Device"):
                opt = DeviceWindowOptimizer(p, prm)
                runs[name] = (lambda o=opt: o.run(poses, codes))
            else:
                err = p.error if "error=" in name else None
                runs[name] = (lambda p=p, err=err: WindowOptimizer(p.layout, p.linearise, prm, solve=p.solve,
                                                                   error=err).run(poses, codes))
        traces, walls = {}, {n: [] for n in runs}
        for name, fn in runs.items():  # warm-up: module loads, allocations, the solver's workspace
            _, _, traces[name] = fn()
        torch.cuda.synchronize()
        for _ in range(reps):
            for name, fn in runs.items():
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                walls[name].append((time.perf_counter() - t0) * 1e6)
        for name, fn in runs.items():
            tr = traces[name]
            print(json.dumps({"case": f"window200 C={cs} ({num_kf} keyframes, {len(pairs)} pairs, {levels} levels "
                                      f"640x480): 10-iteration LM, {name}",
                              "us_total": float(np.median(walls[name])), "us_runs": walls[name],
                              "device_us_total": _device_us(torch, fn, 1), "linearisations": tr.linearisations,
                              "error_evaluations": tr.error_evaluations, "accepted": tr.accepted,
                              "energy_first_last": [tr.energy[0], tr.energy[-1]], "timing": timing}), flush=True)
        del runs, keyframes, shared, jac
        torch.cuda.empty_cache()


def levels_cases(args, torch, print):
    """Coarse to fine against all levels at once.  Every keyframe of the synthetic window holds the same pyramid, so the
    identity poses are the scene's known solution; the starts perturb keyframes 1.. by increasing amounts.  pho_iters =
    4,8,15 has three levels, so the window has three (640x480, 320x240, 160x120); the all-level loop takes as many LM
    steps as the schedule has (30).  Reported per loop: wall time of one run to a synchronise (median of the alternated
    repetitions), summed device time (torch.profiler, separate run), the final pose error against the identity (mean
    translation norm and rotation angle over the keyframes) and the level-0 energy at the final point (the error of the
    level-0 items alone, dfk_window_problem_error under a level-0 mask)."""
    import numpy as np
    from deepfactors_b200 import se3, synth
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import DeviceWindowOptimizer, LMParams, SfmWindowProblem
    sys.path.insert(0, ROOT)
    from bench import window_pairs
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    levels, num_kf, iters = 3, 50, (4, 8, 15)
    steps = sum(i + 1 for i in iters)
    reps = max(3, args.reps // 5)
    timing = ("wall clock of one run() to a synchronise, median over the alternated repetitions; device time = summed "
              "kernel + copy time of one run(), torch.profiler (separate run)")
    for cs in (32, 128):
        base = synth.make_pair(640, 480, cs, levels, seed=7)
        shared = [dict(img=up(L.img0), grad=up(L.grad1), prx_orig=up(L.prx_orig)) for L in base.levels]
        jac = [up(L.prx_jac) for L in base.levels]
        gen = torch.Generator(device="cuda").manual_seed(cs)
        keyframes = [[dict(sh, prx_jac=j + 1e-3 * torch.randn(j.shape, device="cuda", generator=gen),
                           dpt=torch.zeros_like(sh["img"]), valid=torch.zeros_like(sh["img"]))
                      for sh, j in zip(shared, jac)] for _ in range(num_kf)]
        pairs = window_pairs(num_kf, 200)
        cams = [L.cam for L in base.levels]
        al = SfmAligner(cs)
        prm = LMParams(iterations=steps, lambda_init=1e-4)
        probs = {name: SfmWindowProblem(al, cams, keyframes, pairs) for name in ("levels", "all")}
        sched = probs["levels"].level_schedule(iters)
        opts = {"levels": DeviceWindowOptimizer(probs["levels"], prm, schedule=sched),
                "all": DeviceWindowOptimizer(probs["all"], prm)}
        level0 = np.asarray(sched.item_level) == 0
        codes = np.zeros((num_kf, cs))
        for scale in (0.003, 0.01, 0.03):
            rng = np.random.default_rng(int(scale * 1e4))
            poses = np.stack([se3.identity(np.float64)] + [
                se3.make_pose(rng.standard_normal(3) * scale, rng.standard_normal(3) * scale * 3, np.float64)
                for _ in range(num_kf - 1)])
            runs = {n: (lambda o=o: o.run(poses, codes)) for n, o in opts.items()}
            out = {n: fn() for n, fn in runs.items()}  # warm-up, and the result
            torch.cuda.synchronize()
            walls = {n: [] for n in runs}
            for _ in range(reps):
                for n, fn in runs.items():
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    walls[n].append((time.perf_counter() - t0) * 1e6)
            for n, fn in runs.items():
                p, c, tr = out[n]
                dp = opts[n].dev
                dp.set_state(p, c)
                dp.set_active(level0)
                e0 = float(dp.error().cpu()[0])
                dp.set_active(np.ones(dp.num_dense, bool))
                terr = float(np.mean(np.linalg.norm(p[:, 4:], axis=1)))
                rerr = float(np.mean(2.0 * np.arccos(np.clip(np.abs(p[:, 3]), 0.0, 1.0))))
                print(json.dumps({"case": f"window200 C={cs} ({num_kf} keyframes, {len(pairs)} pairs, {levels} levels "
                                          f"640x480), start perturbed by {scale} rad / {3 * scale} m (std): "
                                          + ("pho_iters 4,8,15 (dfk_window_lm_levels)" if n == "levels" else
                                             f"{steps} all-level steps (dfk_window_lm)"),
                                  "us_total": float(np.median(walls[n])), "us_runs": walls[n],
                                  "device_us_total": _device_us(torch, fn, 1), "steps": len(tr.accepted),
                                  "accepted": sum(tr.accepted), "switches": len(tr.switch_energy),
                                  "linearisations": tr.linearisations, "level0_energy": e0,
                                  "mean_translation_error_m": terr, "mean_rotation_error_rad": rerr,
                                  "timing": timing}), flush=True)
        del opts, probs, keyframes, shared, jac
        torch.cuda.empty_cache()


def match_cases(args, torch, print):
    """dfk_reprojection_match_batch against cv2.BFMatcher + the sequential C RANSAC on the host (match_oracle)"""
    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from match_scenes import make_scene

    from deepfactors_b200.aligners import Features, ReprojectionMatchBatch, SfmAligner
    from match_oracle import match_oracle as mo
    try:
        import cv2
        bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    except ImportError:  # the host leg then times the oracle's brute-force matcher instead
        bf = None
    al = SfmAligner(8)
    for name, n, nb, factors in (("connection_orb500", 500, 32, 8), ("connection_brisk1000", 1000, 64, 8),
                                 ("factors64_orb500", 500, 32, 64)):
        scenes = [make_scene(n, 0.4, 0.5, 1000 + j, desc_bytes=nb, max_flips=40) for j in range(factors)]
        items = [dict(query=Features.from_host(sc.kp0, sc.desc0), train=Features.from_host(sc.kp1, sc.desc1),
                      cam=sc.cam, seed=j) for j, sc in enumerate(scenes)]

        def device():
            ReprojectionMatchBatch(al, items)

        wall = _wall_us(torch, device, args.reps)
        dev_us = _device_us(torch, device, args.reps)
        _, counts, ransac = ReprojectionMatchBatch(al, items)
        counts, ransac = counts.cpu().numpy(), ransac.cpu().numpy()
        t0 = time.perf_counter()
        kept = []
        for j, sc in enumerate(scenes):
            if bf is not None:
                ms = bf.match(sc.desc0, sc.desc1)
                m = np.full((n, 2), -1, np.int32)
                for x in ms:
                    m[x.queryIdx] = (x.trainIdx, int(round(x.distance)))
            else:
                m = mo.hamming(sc.desc0, sc.desc1)
            r = mo.reprojection_match(mo.params(sc.cam, seed=j), sc.kp0, sc.desc0, sc.kp1, sc.desc1, m)
            kept.append(len(r.rows))
        host = (time.perf_counter() - t0) * 1e6
        print(json.dumps({"case": f"match_{name}", "factors": factors, "features": n, "descriptor_bytes": nb,
                          "device_wall_us": round(wall, 1), "device_time_us": round(dev_us, 1),
                          "host_us": round(host, 1), "host_matcher": "cv2.BFMatcher" if bf else "oracle",
                          "speedup_wall": round(host / wall, 1),
                          "hypotheses_evaluated_mean": float(ransac[:, 2].mean()),
                          "kept_equal_host": bool(list(counts) == kept)}))


def _kernel_name(key):
    """orb_fast_kernel for 'dfk::(anonymous namespace)::orb_fast_kernel(...)'; other profiler keys as they are"""
    import re
    m = re.search(r"(\w+_kernel)\(", key)
    return m.group(1) if m else key.strip()


def orb_cases(args, torch, print):
    """dfk_orb_detect_batch against cv2.ORB_create(500, 1.2, 1).detectAndCompute on the host, image by image"""
    import numpy as np
    from torch.profiler import ProfilerActivity, profile

    from deepfactors_b200.aligners import OrbDetectBatch, SfmAligner
    try:
        import cv2
    except ImportError:  # no host leg then
        cv2 = None
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from orb_images import images
    z = images()
    al = SfmAligner(8)
    for w, h in ((256, 192), (640, 480)):
        base = [z[f"1047_{w}"], z[f"1052_{w}"]]
        for n in (1, 8, 64):
            rng = np.random.default_rng(n)
            # the two test images, each copy with its own noise so that no two images of a batch are equal
            imgs = [np.clip(base[i % 2].astype(np.int16) + rng.integers(-2, 3, base[0].shape), 0, 255).astype(np.uint8)
                    for i in range(n)]
            dev = [torch.from_numpy(im).cuda() for im in imgs]

            def device():
                OrbDetectBatch(al, dev, 500, 20)

            wall = _wall_us(torch, device, args.reps)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    device()
                torch.cuda.synchronize()
            stages = {e.key: round(e.self_device_time_total / args.reps, 1) for e in prof.key_averages()
                      if e.self_device_time_total > 0}
            dev_us = sum(stages.values())
            counts = OrbDetectBatch(al, dev, 500, 20).counts.cpu().numpy()
            rec = {"case": f"orb_{w}x{h}_x{n}", "images": n, "width": w, "height": h, "nfeatures": 500,
                   "device_wall_us": round(wall, 1), "device_time_us": round(dev_us, 1),
                   "stages_us": {_kernel_name(k): v for k, v in stages.items()}}
            if cv2 is not None:
                orb = cv2.ORB_create(500, 1.2, 1)
                orb.detectAndCompute(imgs[0], None)
                t0 = time.perf_counter()
                host_counts = [len(orb.detectAndCompute(im, None)[0]) for im in imgs]
                host = (time.perf_counter() - t0) * 1e6
                rec.update({"host_us": round(host, 1), "host": f"cv2 {cv2.__version__}, one image at a time",
                            "speedup_wall": round(host / wall, 1), "counts_equal_host": host_counts == list(counts)})
            print(json.dumps(rec))


def orb_pyramid_cases(args, torch, print):
    """dfk_orb_detect_pyramid_batch against the C oracle and cv2.ORB_create(500, 1.2, 8) on the host, image by image"""
    import numpy as np
    from torch.profiler import ProfilerActivity, profile

    from deepfactors_b200.aligners import OrbDetectPyramidBatch, SfmAligner
    try:
        import cv2
    except ImportError:  # no cv2 leg then
        cv2 = None
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from orb_images import images
    from orb_oracle import orb_oracle as oo
    z = images()
    al = SfmAligner(8)
    base = [z["1047_640"], z["1052_640"]]
    for n in (1, 8, 64):
        rng = np.random.default_rng(n)
        imgs = [np.clip(base[i % 2].astype(np.int16) + rng.integers(-2, 3, base[0].shape), 0, 255).astype(np.uint8)
                for i in range(n)]
        dev = [torch.from_numpy(im).cuda() for im in imgs]

        def device():
            OrbDetectPyramidBatch(al, dev, 500, 1.2, 8, 20)

        wall = _wall_us(torch, device, args.reps)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                device()
            torch.cuda.synchronize()
        stages = {}
        for e in prof.key_averages():
            if e.self_device_time_total > 0:
                k = _kernel_name(e.key)
                stages[k] = round(stages.get(k, 0.0) + e.self_device_time_total / args.reps, 1)
        dev_us = sum(stages.values())
        counts = OrbDetectPyramidBatch(al, dev, 500, 1.2, 8, 20).counts.cpu().numpy()
        t0 = time.perf_counter()
        oracle_counts = [oo.detect_pyramid(im, 500, 1.2, 8, 20, 1000).count for im in imgs]
        oracle_us = (time.perf_counter() - t0) * 1e6
        rec = {"case": f"orb_pyramid_640x480_x{n}", "images": n, "width": 640, "height": 480, "nfeatures": 500,
               "scale_factor": 1.2, "nlevels": 8, "device_wall_us": round(wall, 1), "device_time_us": round(dev_us, 1),
               "stages_us": stages, "host_oracle_us": round(oracle_us, 1),
               "counts_equal_oracle": oracle_counts == list(counts)}
        if cv2 is not None:
            orb = cv2.ORB_create(500, 1.2, 8)
            orb.detectAndCompute(imgs[0], None)
            t0 = time.perf_counter()
            host_counts = [len(orb.detectAndCompute(im, None)[0]) for im in imgs]
            host = (time.perf_counter() - t0) * 1e6
            rec.update({"host_us": round(host, 1), "host": f"cv2 {cv2.__version__}, one image at a time",
                        "speedup_wall": round(host / wall, 1), "counts_equal_host": host_counts == list(counts)})
        print(json.dumps(rec))


def _full_voc(k: int, L: int, D: int, seed: int) -> dict:
    """a complete k-ary tree of depth L listed breadth first, random centroids, leaf weights in (0.1, 3)"""
    import numpy as np
    rng = np.random.default_rng(seed)
    sizes = [k ** d for d in range(1, L + 1)]
    N = sum(sizes)
    ids = np.arange(1, N + 1, dtype=np.int64)
    parents = np.zeros(N, np.int64)
    first = 0
    for d, n in enumerate(sizes):
        if d:
            parents[first:first + n] = (first - sizes[d - 1]) + np.arange(n) // k + 1
        first += n
    leaves = ids[N - sizes[-1]:]
    w = np.zeros(N)
    w[N - sizes[-1]:] = rng.uniform(0.1, 3.0, sizes[-1])
    return dict(k=k, L=L, weighting=0, scoring=0, descriptor_bytes=D, node_ids=ids.astype(np.int32),
                parent_ids=parents.astype(np.int32), weights=w, descriptors=rng.integers(0, 256, (N, D), np.uint8),
                word_ids=np.arange(len(leaves), dtype=np.int32), word_nodes=leaves.astype(np.int32))


def bow_cases(args, torch, print):
    """dfk_bow_transform_batch and dfk_bow_database_query_batch against the sequential C oracle on one host thread"""
    import numpy as np

    from bow_oracle import bow_oracle as bo
    from deepfactors_b200 import aligners as A
    vocs = {"small_voc": A.load_dbow2_vocabulary(os.path.join(ROOT, "tests", "golden", "dbow2_small_voc.yml.gz")),
            "k10_L6": _full_voc(10, 6, 32, 0)}
    for name, v in vocs.items():
        gv, ov = A.BowVocabulary(v), bo.Vocabulary(v)
        D = v["descriptor_bytes"]
        for n in (1, 8, 64):
            rng = np.random.default_rng(n)
            sets = [rng.integers(0, 256, (500, D), np.uint8) for _ in range(n)]
            dev = [torch.from_numpy(s).cuda() for s in sets]
            fn = lambda: A.BowTransformBatch(gv, dev)
            wall = _wall_us(torch, fn, args.reps)
            dus = _device_us(torch, fn, args.reps)
            t0 = time.perf_counter()
            for s in sets:
                ov.transform(s)
            host = (time.perf_counter() - t0) * 1e6
            print(json.dumps({"case": "bow_transform", "vocabulary": name, "words": len(v["word_ids"]), "frames": n,
                              "features": 500, "device_wall_us": round(wall, 1), "device_us": round(dus, 1),
                              "oracle_host_us": round(host, 1), "speedup_wall": round(host / wall, 1)}))
    v = vocs["small_voc"]
    gv, ov = A.BowVocabulary(v), bo.Vocabulary(v)
    rng = np.random.default_rng(7)
    images = [rng.integers(0, 256, (500, 48), np.uint8) for _ in range(100)]
    b = A.BowTransformBatch(gv, [torch.from_numpy(s).cuda() for s in images])
    vecs, ovecs = b.vectors(), [ov.transform(s)[1:] for s in images]
    q = rng.integers(0, 256, (500, 48), np.uint8)
    qv = A.BowTransformBatch(gv, [torch.from_numpy(q).cuda()]).vectors()
    qo = ov.transform(q)[1:]
    for entries in (100, 1000, 10000):
        db, odb = A.BowDatabase(gv), bo.Database()
        for s in range(0, entries, 100):
            db.add(vecs[:min(100, entries - s)])
        for e in range(entries):
            odb.add(*ovecs[e % 100])
        fn = lambda: db.query(qv, 20)
        wall = _wall_us(torch, fn, args.reps)
        dus = _device_us(torch, fn, args.reps)
        t0 = time.perf_counter()
        odb.query(*qo, 20)
        host = (time.perf_counter() - t0) * 1e6
        print(json.dumps({"case": "bow_query", "entries": entries, "max_results": 20, "device_wall_us": round(wall, 1),
                          "device_us": round(dus, 1), "oracle_host_us": round(host, 1),
                          "speedup_wall": round(host / wall, 1)}))


def preprocess_cases(args, torch, print):
    """dfk_preprocess_batch against cv2.remap + cvtColor + convertTo on the host, frame by frame"""
    import numpy as np
    from torch.profiler import ProfilerActivity, profile

    import ctypes

    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import PreprocessBatch, SfmAligner, resize_viewport
    from deepfactors_b200.synth import Camera
    cam4 = lambda c: (c.fx, c.fy, c.u0, c.v0)
    try:
        import cv2
    except ImportError:  # no host leg then
        cv2 = None
    z = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_frames.npz"))
    base = [np.repeat(np.repeat(z[f"image_{k}"], 2, axis=0), 2, axis=1) for k in ("1047", "1052")]
    src_cam = resize_viewport(Camera(525.0, 525.0, 319.5, 239.5, 640.0, 480.0), 640, 480)
    out_cam = Camera.scenenet(256, 192)
    levels = 4
    al = SfmAligner(8)
    for n in (1, 8, 64):
        rng = np.random.default_rng(n)
        frames = [np.clip(base[i % 2].astype(np.int16) + rng.integers(-2, 3, base[0].shape), 0, 255).astype(np.uint8)
                  for i in range(n)]
        dev = [torch.from_numpy(f).cuda() for f in frames]

        def device():
            PreprocessBatch(al, dev, src_cam, out_cam, levels)

        wall = _wall_us(torch, device, args.reps)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                device()
            torch.cuda.synchronize()
        stages = {e.key: round(e.self_device_time_total / args.reps, 1) for e in prof.key_averages()
                  if e.self_device_time_total > 0}
        # the C call alone: output buffers and items built once, as a caller that keeps its buffers does
        outs = PreprocessBatch(al, dev, src_cam, out_cam, levels)
        keep, items = [], []
        for f, o in zip(dev, outs):
            la = (_lib.DfkImage * levels)(*[_lib.DfkImage(t.data_ptr(), 4 * t.shape[1], t.shape[1], t.shape[0])
                                            for t in o.levels])
            ga = (_lib.DfkImage * levels)(*[_lib.DfkImage(t.data_ptr(), 8 * t.shape[1], t.shape[1], t.shape[0])
                                            for t in o.grads])
            keep += [la, ga]
            items.append(_lib.DfkPreprocessItem(
                _lib.DfkImage(f.data_ptr(), 3 * 640, 640, 480), _lib.DfkCamera(*cam4(src_cam), 640, 480),
                _lib.DfkCamera(*cam4(out_cam), 256, 192), _lib.DfkImage(o.color.data_ptr(), 3 * 256, 256, 192),
                _lib.DfkImage(o.gray.data_ptr(), 256, 256, 192), ctypes.cast(la, ctypes.POINTER(_lib.DfkImage)),
                ctypes.cast(ga, ctypes.POINTER(_lib.DfkImage)), 0))
        arr = (_lib.DfkPreprocessItem * n)(*items)
        L = _lib.lib()

        def c_call():
            _lib.check(al._hd.h, L.dfk_preprocess_batch(al._hd.h, arr, n, levels, None))

        c_wall = _wall_us(torch, c_call, args.reps)
        rec = {"case": f"preprocess_640x480_to_256x192_x{n}", "frames": n, "levels": levels, "grads": True,
               "device_wall_us": round(wall, 1), "c_call_wall_us": round(c_wall, 1),
               "device_time_us": round(sum(stages.values()), 1),
               "stages_us": {_kernel_name(k): v for k, v in stages.items()}}
        if cv2 is not None:
            K = lambda c: np.array([[c.fx, 0, c.u0], [0, c.fy, c.v0], [0, 0, 1]], np.float64)
            m1, m2 = cv2.initUndistortRectifyMap(K(src_cam), None, None, K(out_cam), (256, 192), cv2.CV_32FC1)

            def host_chain(f):
                gray = cv2.cvtColor(cv2.remap(f, m1, m2, cv2.INTER_LINEAR), cv2.COLOR_RGB2GRAY)
                # cv2's Python API has no convertTo; this numpy fp32 product is bitwise what convertTo(CV_32FC1,
                # 1 / 255.0) gives
                return gray.astype(np.float32) * np.float32(1.0 / 255.0)

            host_chain(frames[0])
            t0 = time.perf_counter()
            for f in frames:
                host_chain(f)
            host = (time.perf_counter() - t0) * 1e6
            rec.update({"host_us": round(host, 1), "host_levels": 0,
                        "host": f"cv2 {cv2.__version__} remap + cvtColor, then a numpy fp32 product (bitwise convertTo), "
                                "one frame at a time, no pyramid",
                        "speedup_wall": round(host / wall, 1)})
        print(json.dumps(rec))


def solve_fill(K, links):
    """(tiles, fp64 flops) of the block Cholesky of a window whose keyframes are joined by `links`, eliminated in index
    order (the symbolic analysis of dfk_window_solver_create): per column with n off-diagonal tiles, the diagonal
    factor B^3 / 3, n triangular solves B^3 and n (n + 1) / 2 Schur updates 2 B^3, in units of B^3"""
    below = [set() for _ in range(K)]
    for a, b in links:
        if a != b:
            below[min(a, b)].add(max(a, b))
    units = 0.0
    for j in range(K):
        rows = sorted(below[j])
        for x in range(len(rows)):
            for y in range(x):
                below[rows[y]].add(rows[x])
        n = len(rows)
        units += 1.0 / 3.0 + n + n * (n + 1)
    return K + sum(len(r) for r in below), units


def solve_cases(args, torch, print):
    import numpy as np
    from bench import window_pairs
    from deepfactors_b200.aligners import SfmAligner, Window, WindowSolver
    from deepfactors_b200.window_opt import damped_solve
    for name, K, P, cs in (("window200", 50, 200, 32), ("window200", 50, 200, 128), ("ba2k", 200, 2000, 32)):
        pairs = window_pairs(K, P)
        al = SfmAligner(cs)
        win = Window(al, K, pairs, list(range(P)), [(0, 0)] * P)
        lay = win.layout
        NP = 12 + cs
        rng = np.random.default_rng(1)
        JtJ = np.empty((P, NP, NP), np.float32)
        Jtr = np.empty((P, NP), np.float32)
        for p in range(P):  # random Gram records: every block positive definite
            A = rng.standard_normal((2 * NP, NP + 1)).astype(np.float32)
            JtJ[p] = A[:, :NP].T @ A[:, :NP]
            Jtr[p] = A[:, :NP].T @ A[:, NP]
        buf = torch.from_numpy(lay.pack(list(range(P)), JtJ, Jtr, np.ones(P, np.float32), np.zeros(P), [(0, 0)] * P)).cuda()
        fixed = tuple(range(6))
        lam = 1e-4
        sol = WindowSolver(win, fixed)
        B = lay.B
        tiles, units = solve_fill(K, pairs)
        assert tiles == sol.tiles
        flops = units * B ** 3

        def run_torch():
            H, g, _, _ = lay.to_dense(buf)
            dx = damped_solve(H, g, lam, fixed)
            torch.cuda.synchronize()
            return dx

        def run_dev():
            dx, info = sol.solve(buf, lam)
            torch.cuda.synchronize()
            return dx, info

        ref = run_torch()
        dx, info = run_dev()
        assert int(info.item()) == 0
        err = float((dx - ref).abs().max() / ref.abs().max())
        reps = min(args.reps, 5) if K > 100 else args.reps
        tt, td = [], []
        for _ in range(reps):  # alternated
            t0 = time.perf_counter(); run_torch(); tt.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); run_dev(); td.append(time.perf_counter() - t0)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run_dev()
        ev = [e for e in prof.events() if e.device_type.name == "CUDA" and "window_solve" in e.name]
        dev_ms = sum(e.device_time for e in ev) / 1e3
        per = {}
        for e in ev:
            k = e.name.split("window_solve_")[1].split("_kernel")[0]
            per[k] = per.get(k, 0.0) + e.device_time / 1e3
        print(json.dumps(dict(
            case="window_solve", shape=name, K=K, pairs=P, C=cs, tiles=tiles, dense_tiles=K * (K + 1) // 2,
            factor_mb=round((tiles + K) * B * B * 8 / 1e6, 1), dense_mb=round((K * B) ** 2 * 8 / 1e6, 1),
            torch_ms_median=round(1e3 * float(np.median(tt)), 3), torch_ms_min=round(1e3 * min(tt), 3),
            device_ms_median=round(1e3 * float(np.median(td)), 3), device_ms_min=round(1e3 * min(td), 3),
            device_kernel_ms=round(dev_ms, 3), kernel_ms_by_kind={k: round(v, 3) for k, v in per.items()},
            launches=len(ev), fill_gflop=round(flops / 1e9, 2), fp64_tflops=round(flops / (dev_ms * 1e-3) / 1e12, 3),
            rel_diff_vs_torch=err, reps=reps)))


def mesh_cases(args, torch, print):
    """dfk_keyframe_mesh_batch from the depth and from the fused decode (C = 32) against the sequential C oracle"""
    import ctypes
    import numpy as np
    from torch.profiler import ProfilerActivity, profile

    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import KeyframeMeshParams, SfmAligner
    from mesh_oracle import mesh_oracle as mo
    cs = 32
    al = SfmAligner(cs)
    prm = KeyframeMeshParams()
    cparams = prm.to_c()
    L = _lib.lib()
    for w, h in ((256, 192), (640, 480)):
        ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
        for n in (1, 8, 64):
            rng = np.random.default_rng(n)
            items = (_lib.DfkKeyframeMeshItem * n)()
            keep, host = [], []
            for i in range(n):
                prx = (0.5 + 0.1 * np.sin(xs / 17.0 + i) * np.cos(ys / 13.0)).astype(np.float32)
                jac = (rng.standard_normal((h, w, cs)) * 1e-3).astype(np.float32)
                std = rng.uniform(-2.0, 0.5, (h, w)).astype(np.float32)  # below the noise threshold: a dense mesh
                col = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
                code = np.zeros(cs, np.float32)
                t = {k: torch.from_numpy(v).cuda() for k, v in dict(prx=prx, jac=jac, std=std, col=col).items()}
                t["vld"] = torch.ones((h, w), dtype=torch.float32, device="cuda")
                t["dpt"] = torch.empty((h, w), dtype=torch.float32, device="cuda")
                t["u16"] = torch.empty((h, w), dtype=torch.int16, device="cuda")
                keep += [t, code]
                a = items[i]
                a.std = _lib.DfkImage(t["std"].data_ptr(), 4 * w, w, h)
                a.valid = _lib.DfkImage(t["vld"].data_ptr(), 4 * w, w, h)
                a.color = _lib.DfkImage(t["col"].data_ptr(), 3 * w, w, h)
                a.cam = _lib.DfkCamera(0.9 * w, 0.9 * w, w / 2 - 0.5, h / 2 - 0.5, w, h)
                a.pose_wk = (ctypes.c_float * 7)(0.01 * i, 0.0, 0.0, 1.0, 0.1 * i, 0.0, 0.0)
                a.vertex_capacity, a.triangle_capacity = w * h, 2 * w * h
                a.depth_u16 = _lib.DfkImage(t["u16"].data_ptr(), 2 * w, w, h)
                host.append(dict(std=std, col=col, cam=(0.9 * w, 0.9 * w, w / 2 - 0.5, h / 2 - 0.5),
                                 pose=np.frombuffer(a.pose_wk, np.float32).copy()))
            # the decoded depths, by dfk_update_depth_batch, for the depth path and the oracle
            dec = (_lib.DfkDepthDecodeItem * n)()
            for i in range(n):
                t = keep[2 * i]
                dec[i].prx_orig = _lib.DfkImage(t["prx"].data_ptr(), 4 * w, w, h)
                dec[i].prx_jac = _lib.DfkImage(t["jac"].data_ptr(), 4 * w * cs, w, h)
                dec[i].dpt = _lib.DfkImage(t["dpt"].data_ptr(), 4 * w, w, h)
                dec[i].code = keep[2 * i + 1].ctypes.data_as(ctypes.POINTER(ctypes.c_float))
            al._hd.use_torch_stream()
            _lib.check(al._hd.h, L.dfk_update_depth_batch(al._hd.h, dec, n, cs))
            V, T = n * w * h, 2 * n * w * h
            out = [torch.empty((V, 3), device="cuda"), torch.empty((V, 3), device="cuda"),
                   torch.empty((V, 3), dtype=torch.uint8, device="cuda"), torch.empty(V, dtype=torch.int32, device="cuda"),
                   torch.empty((T, 3), dtype=torch.int32, device="cuda"),
                   torch.empty((n, 2), dtype=torch.int32, device="cuda")]
            ptrs = [ctypes.c_void_p(o.data_ptr()) for o in out]
            for source in ("depth", f"decode_c{cs}"):
                for i in range(n):
                    t, a = keep[2 * i], items[i]
                    if source == "depth":
                        a.dpt = _lib.DfkImage(t["dpt"].data_ptr(), 4 * w, w, h)
                        a.prx_orig = a.prx_jac = _lib.DfkImage()
                        a.code = None
                    else:
                        a.dpt = _lib.DfkImage()
                        a.prx_orig, a.prx_jac, a.code = dec[i].prx_orig, dec[i].prx_jac, dec[i].code

                def call():
                    _lib.check(al._hd.h, L.dfk_keyframe_mesh_batch(al._hd.h, items, n, cs, ctypes.byref(cparams),
                                                                    *ptrs))

                wall = _wall_us(torch, call, args.reps)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.reps):
                        call()
                    torch.cuda.synchronize()
                stages = {_kernel_name(e.key): round(e.self_device_time_total / args.reps, 1) for e in prof.key_averages()
                          if e.self_device_time_total > 0}
                dev_us = sum(stages.values())
                counts = out[5].cpu().numpy().astype(np.int64)
                nv, nt = int(counts[:, 0].sum()), int(counts[:, 1].sum())
                # algorithmic bytes: every input pixel read once (depth or proximity + C Jacobian floats, log-stdev,
                # validity, colour), the uint16 depth written, and the rows (position, normal, colour, pixel; triangle)
                px = n * w * h
                src = 4 * px if source == "depth" else 4 * px * (1 + cs)
                nbytes = src + px * (4 + 4 + 3 + 2) + nv * (12 + 12 + 3 + 4) + nt * 12
                rec = {"case": f"keyframe_mesh_{w}x{h}_x{n}_{source}", "keyframes": n, "vertices": nv, "triangles": nt,
                       "wall_us": round(wall, 1), "device_time_us": round(dev_us, 1), "stages_us": stages,
                       "algorithmic_bytes": nbytes,
                       "achieved_gbs": round(nbytes / (dev_us * 1e-6) / 1e9, 1) if dev_us > 0 else "not measured"}
                if source == "depth":
                    dpt = [keep[2 * i]["dpt"].cpu().numpy() for i in range(n)]
                    t0 = time.perf_counter()
                    for i in range(n):
                        hd = host[i]
                        mo.mesh(dpt[i], hd["cam"], hd["pose"], std=hd["std"], vld=np.ones((h, w), np.float32),
                                color=hd["col"])
                    rec["oracle_host_us"] = round((time.perf_counter() - t0) * 1e6, 1)
                    rec["oracle_threads"] = 1
                else:
                    rec["oracle_host_us"] = "not measured (the oracle takes a decoded depth)"
                print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
