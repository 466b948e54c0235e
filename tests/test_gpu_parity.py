"""GPU parity tests: the CUDA path (through the C ABI of libdfk.so) against the CPU oracle.

Bars (BASELINE.md section 4, from the reference's own tests):
  * inlier counts EXACTLY equal to the CPU path           (tests/ut_sfmaligner.cpp:320)
  * JtJ entries: the reference accepts 1e-1 absolute GPU-vs-CPU on entries up to ~1e4-1e5, i.e.
    ~1e-5 of max|H| (ut_sfmaligner.cpp:324-326).  We state the fp32 tolerance against the fp64 oracle:
        max |H_gpu - H_f64| <= 2e-5 * max|H_f64|        (fp32 Gram path)
    and report next to it the same figure for the oracle's own fp32 flavour (the reference-like CPU
    path), which is of the same order.
  * Jtr: 1e-4 * max|Jtr| ; residual: 1e-5 relative.
Sizes are those the oracle finishes in seconds (160x120/C=8 = BASELINE configs[0], 320x240/C=32,
one 640x480/C=32 level); full-size properties are in test_gpu_properties.py.
"""
import numpy as np
import pytest

from deepfactors_b200 import se3, synth

pytestmark = pytest.mark.gpu

H_TOL = 2e-5
JTR_TOL = 1e-4
RES_TOL = 1e-5


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def pitched(torch, arr, extra_px=0):
    """upload a host array [H, W(, K)] into a device buffer whose rows are padded (pitch != width)"""
    a = np.ascontiguousarray(arr, dtype=np.float32)
    h, w = a.shape[:2]
    k = a.shape[2] if a.ndim == 3 else 1
    row = (w + extra_px) * k
    buf = torch.zeros((h, row), dtype=torch.float32, device="cuda")
    buf[:, :w * k] = torch.from_numpy(a.reshape(h, w * k)).cuda()
    if a.ndim == 2:
        return buf[:, :w]
    return torch.as_strided(buf, (h, w, k), (row, k, 1))


def upload_level(torch, L, extra_px=0):
    d = dict(img0=pitched(torch, L.img0, extra_px), img1=pitched(torch, L.img1, extra_px),
             dpt0=pitched(torch, L.dpt0, extra_px), std0=pitched(torch, L.std0, extra_px),
             prx0_jac=pitched(torch, L.prx_jac, extra_px), grad1=pitched(torch, L.grad1, extra_px),
             prx_orig=pitched(torch, L.prx_orig, extra_px))
    d["valid0"] = pitched(torch, np.zeros_like(L.img0), extra_px)
    return d


def compare_step(gpu, o32, o64, what):
    # the bar of tests/ut_sfmaligner.cpp:320: inliers equal to the fp32 CPU path, exactly
    assert gpu.inliers == o32.inliers, f"{what}: inliers gpu={gpu.inliers} cpu_fp32={o32.inliers}"
    if o64.inliers != o32.inliers:
        # fp32 rounding moves pixels that sit exactly on the validity border (e.g. identity pose): the fp64
        # truth then sums a different pixel set, so compare against the fp32 CPU path instead
        print(f"{what}: fp64 oracle has {o64.inliers} inliers vs {o32.inliers} in fp32 -- comparing to fp32")
        H32 = o32.dense().astype(np.float64)
        Hg = gpu.toDenseMatrix().astype(np.float64)
        assert np.abs(Hg - H32).max() <= 2 * H_TOL * np.abs(H32).max(), what
        assert abs(gpu.residual - o32.residual) <= 2 * RES_TOL * o32.residual, what
        return
    H64 = o64.dense()
    Hg = gpu.toDenseMatrix().astype(np.float64)
    scale = np.abs(H64).max()
    err_gpu = np.abs(Hg - H64).max() / scale
    err_cpu32 = np.abs(o32.dense().astype(np.float64) - H64).max() / scale
    print(f"{what}: max|H-H64|/max|H64| gpu={err_gpu:.2e} cpu_fp32={err_cpu32:.2e}; max|H|={scale:.3e}")
    assert err_gpu <= H_TOL, f"{what}: H error {err_gpu:.3e}"
    jscale = np.abs(o64.Jtr).max()
    assert np.abs(gpu.Jtr - o64.Jtr).max() <= JTR_TOL * jscale, what
    assert abs(gpu.residual - o64.residual) <= RES_TOL * o64.residual, what
    assert np.allclose(Hg, Hg.T)


@pytest.mark.parametrize("w,h,cs,extra", [(160, 120, 8, 0), (160, 120, 8, 12), (320, 240, 32, 0), (320, 240, 32, 20),
                                          (640, 480, 32, 0), (200, 96, 16, 4), (202, 96, 8, 1),
                                          # the coarse pyramid levels of the benchmark workload, on their own
                                          (160, 120, 32, 0), (80, 60, 32, 4),
                                          # the code sizes the reference declares but cannot launch
                                          # (cu_sfmaligner.cpp:170-173,210-211); BASELINE config C=128
                                          (160, 120, 64, 0), (202, 96, 64, 1), (160, 120, 128, 4), (320, 240, 128, 0)])
def test_sfm_run_step_matches_oracle(torch_mod, oracle, w, h, cs, extra):
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner, SfmAlignerParams, DenseSfmParams
    pair = synth.make_pair(w, h, cs, 1, seed=w + cs, code_sigma=0.5)
    L = pair.levels[0]
    dev = upload_level(torch, L, extra)
    modes = ("fp32", "tf32x3") if cs == 32 else ("fp32",)
    # production / reference-test Huber thresholds (dense_sfm.h:38, ut_sfmaligner.cpp:69) x Gram engines
    for delta, mode in [(d, m) for d in (0.1, 0.5) for m in modes]:
        dev["valid0"].zero_()
        al = SfmAligner(cs, SfmAlignerParams(sfmparams=DenseSfmParams(huber_delta=delta)), gram_mode=mode)
        g = al.RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"], dev["img1"], dev["dpt0"], dev["std0"],
                       dev["valid0"], dev["prx0_jac"], dev["grad1"])
        prm = oracle.default_params(huber_delta=delta)
        v_cpu = np.zeros((h, w), dtype=np.float32)
        o32 = oracle.sfm_run_step(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, v_cpu, L.prx_jac, L.grad1, prm,
                                  precision="f32")
        o64 = oracle.sfm_run_step(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, None, L.prx_jac, L.grad1, prm,
                                  precision="f64")
        compare_step(g, o32, o64, f"{w}x{h} C={cs} pitch+{extra} delta={delta} gram={mode}")
        # valid0 side effect: exactly the oracle's mask
        v_gpu = dev["valid0"].cpu().numpy()
        assert np.array_equal(v_gpu, v_cpu)


def test_sfm_identity_pose_all_pixels_inliers(torch_mod, oracle):
    """worst-case work: identity relative pose -> every interior pixel is an inlier"""
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    pair = synth.make_pair(320, 240, 32, 1, seed=5, identity_pose=True)
    L = pair.levels[0]
    dev = upload_level(torch, L)
    o32 = oracle.sfm_run_step(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, None, L.prx_jac, L.grad1)
    o64 = oracle.sfm_run_step(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, None, L.prx_jac, L.grad1,
                              precision="f64")
    for mode in ("fp32", "tf32x3"):
        al = SfmAligner(32, gram_mode=mode)
        g = al.RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"], dev["img1"], dev["dpt0"], None,
                       dev["valid0"], dev["prx0_jac"], dev["grad1"])
        assert abs(g.inliers - (320 - 4) * (240 - 4)) <= 2 * (320 + 240)  # up to rounding on the border rows/cols
        compare_step(g, o32, o64, f"identity gram={mode}")


@pytest.mark.parametrize("w,h,cs", [(33, 7, 32), (5, 5, 8), (64, 5, 32), (129, 6, 16), (12, 9, 64), (257, 5, 128)])
def test_sfm_degenerate_image_sizes(torch_mod, oracle, w, h, cs):
    """ragged / tiny inputs: fewer pixels than one tile, rows shorter than a TMA segment, odd widths (cooperative
    staging instead of bulk copies), items that give most CTAs nothing to do"""
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    pair = synth.make_pair(w, h, cs, 1, seed=w * h, identity_pose=True)
    L = pair.levels[0]
    dev = upload_level(torch, L, extra_px=1)
    v_cpu = np.zeros((h, w), dtype=np.float32)
    o32 = oracle.sfm_run_step(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, v_cpu, L.prx_jac, L.grad1)
    o64 = oracle.sfm_run_step(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, None, L.prx_jac, L.grad1,
                              precision="f64")
    for mode in (("fp32", "tf32x3") if cs == 32 else ("auto",)):
        dev["valid0"].zero_()
        al = SfmAligner(cs, gram_mode=mode)
        g = al.RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"], dev["img1"], dev["dpt0"], None,
                       dev["valid0"], dev["prx0_jac"], dev["grad1"])
        assert g.inliers == o32.inliers == int(v_cpu.sum())
        assert np.array_equal(dev["valid0"].cpu().numpy(), v_cpu)
        if o32.inliers:
            compare_step(g, o32, o64, f"{w}x{h} C={cs} gram={mode}")
        else:
            assert g.residual == 0.0 and not np.any(g.JtJ)


def test_sfm_batch_of_mixed_sizes_matches_single_calls(torch_mod):
    """one launch over items of very different sizes (a 320x240 level next to 7-row and 5x5 images) == per-item calls"""
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(32)
    items, singles = [], []
    for k, (w, h) in enumerate([(320, 240), (33, 7), (5, 5), (160, 120), (64, 5), (31, 33)]):
        pair = synth.make_pair(w, h, 32, 1, seed=60 + k, identity_pose=(k % 2 == 1))
        L = pair.levels[0]
        dev = upload_level(torch, L)
        items.append(dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, **{k2: dev[k2] for k2 in (
            "img0", "img1", "dpt0", "valid0", "prx0_jac", "grad1")}))
        singles.append(al.RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"], dev["img1"], dev["dpt0"], None,
                                  dev["valid0"], dev["prx0_jac"], dev["grad1"]))
    recs = al.unpack(al.RunStepBatch(al.make_work_items(items)))
    for got, ref in zip(recs, singles):
        assert got.inliers == ref.inliers
        scale = max(np.abs(ref.JtJ).max(), 1e-30)
        assert np.abs(got.JtJ - ref.JtJ).max() <= 1e-5 * scale
        assert abs(got.residual - ref.residual) <= 1e-5 * max(ref.residual, 1e-12)


def test_sfm_no_overlap_gives_zero_system(torch_mod):
    """zero overlap: inliers == 0, zero Hessian (photometric_factor.cpp:279-282 then sets residual = inf)"""
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    pair = synth.make_pair(160, 120, 8, 1, seed=1)
    L = pair.levels[0]
    dev = upload_level(torch, L)
    pose1 = se3.make_pose([0, 0, 0], [0, 0, 100.0])  # camera 1 far in front: every point lands behind it
    al = SfmAligner(8, gram_mode="fp32")
    g = al.RunStep(pair.pose0, pose1, pair.code, L.cam, dev["img0"], dev["img1"], dev["dpt0"], None, dev["valid0"],
                   dev["prx0_jac"], dev["grad1"])
    assert g.inliers == 0 and g.residual == 0.0
    assert not np.any(g.JtJ) and not np.any(g.Jtr)
    assert float(dev["valid0"].abs().sum()) == 0.0


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_sfm_batch_matches_single_calls_and_is_deterministic(torch_mod, mode):
    """a 4-level pyramid of 2 pairs in ONE launch == the per-level calls, bit for bit across runs"""
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(32, gram_mode=mode)
    items, singles = [], []
    for s in range(2):
        pair = synth.make_pair(320, 240, 32, 4, seed=20 + s, code_sigma=0.3, phase=0.2 * s)
        for L in pair.levels:
            dev = upload_level(torch, L)
            items.append(dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, **{k: dev[k] for k in (
                "img0", "img1", "dpt0", "valid0", "prx0_jac", "grad1")}))
            singles.append(al.RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"], dev["img1"], dev["dpt0"],
                                      None, dev["valid0"], dev["prx0_jac"], dev["grad1"]))
    work = al.make_work_items(items)
    rec1 = al.RunStepBatch(work).clone()
    rec2 = al.RunStepBatch(work).clone()
    torch.cuda.synchronize()
    assert torch.equal(rec1, rec2), "batched launch is not bitwise reproducible"
    for got, ref in zip(al.unpack(rec1), singles):
        assert got.inliers == ref.inliers
        scale = np.abs(ref.JtJ).max()
        # different CTA partition => different summation grouping, same math
        assert np.abs(got.JtJ - ref.JtJ).max() <= 1e-5 * scale
        assert abs(got.residual - ref.residual) <= 1e-5 * max(ref.residual, 1e-12)


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_sfm_sm_limit_changes_the_grid_not_the_result(torch_mod, mode):
    """dfk_set_sm_limit (SMs left to a concurrent collective): same inliers, same sums up to the summation grouping,
    bitwise reproducible for a given limit, and 0 restores the full grid"""
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(32, gram_mode=mode)
    pair = synth.make_pair(640, 480, 32, 3, seed=31, code_sigma=0.3)
    items = []
    for L in pair.levels:
        dev = upload_level(torch, L)
        items.append(dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, **{k: dev[k] for k in (
            "img0", "img1", "dpt0", "valid0", "prx0_jac", "grad1")}))
    work = al.make_work_items(items)
    full = al.RunStepBatch(work).clone()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for limit in (sms - 4, 7, 1):
        al.SetSmLimit(limit)
        a = al.RunStepBatch(work).clone()
        b = al.RunStepBatch(work).clone()
        torch.cuda.synchronize()
        assert torch.equal(a, b), f"limit {limit}: not bitwise reproducible"
        for got, ref in zip(al.unpack(a), al.unpack(full)):
            assert got.inliers == ref.inliers
            assert np.abs(got.JtJ - ref.JtJ).max() <= 1e-5 * np.abs(ref.JtJ).max()
            assert abs(got.residual - ref.residual) <= 1e-5 * max(ref.residual, 1e-12)
    al.SetSmLimit(0)
    assert torch.equal(al.RunStepBatch(work), full)
    with pytest.raises(Exception):
        al.SetSmLimit(-1)


@pytest.mark.parametrize("cs,w,h,mode", [(32, 320, 240, "auto"), (32, 320, 240, "fp32"), (8, 160, 120, "auto"),
                                         (16, 200, 96, "auto"), (64, 160, 120, "auto"), (128, 160, 120, "auto"),
                                         (32, 202, 96, "auto")])
def test_sfm_fused_depth_decode_equals_update_depth_then_run_step(torch_mod, oracle, cs, w, h, mode):
    """PhotometricFactor::UpdateDepthMaps + RunAlignmentStep (photometric_factor.cpp:229,331-341) in ONE launch: the
    decoded depth map and the result records are bit-identical to UpdateDepth followed by RunStep, and the depth agrees
    with the CPU DepthFromCode (warping.h:30-69) to rounding."""
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner, UpdateDepth
    levels = 2
    pair = synth.make_pair(w, h, cs, levels, seed=40 + cs, code_sigma=0.3)
    al = SfmAligner(cs, gram_mode=mode)
    two_step, fused = [], []
    keep = []
    for L in pair.levels:
        dev = upload_level(torch, L, extra_px=0 if w % 4 else 4)
        dpt_a = torch.zeros_like(dev["dpt0"])
        UpdateDepth(pair.code, dev["prx_orig"], dev["prx0_jac"], 2.0, dpt_a)
        dpt_b = torch.full_like(dev["dpt0"], -7.0)  # must be overwritten everywhere by the fused launch
        va, vb = torch.zeros_like(dev["valid0"]), torch.zeros_like(dev["valid0"])
        base = dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, img0=dev["img0"], img1=dev["img1"],
                    prx0_jac=dev["prx0_jac"], grad1=dev["grad1"])
        two_step.append(dict(base, dpt0=dpt_a, valid0=va))
        fused.append(dict(base, dpt0=dpt_b, valid0=vb, prx_orig=dev["prx_orig"], code=pair.code))
        keep.append((dev, dpt_a, dpt_b, va, vb, L))
    rec_a = al.RunStepBatch(al.make_work_items(two_step)).clone()
    rec_b = al.RunStepBatch(al.make_work_items(fused)).clone()
    torch.cuda.synchronize()
    for dev, dpt_a, dpt_b, va, vb, L in keep:
        assert torch.equal(dpt_a, dpt_b), "decoded depth differs from UpdateDepth"
        assert torch.equal(va, vb)
        ref = oracle.update_depth(pair.code, L.prx_orig, L.prx_jac, 2.0)
        got = dpt_b.cpu().numpy()
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()
    assert torch.equal(rec_a, rec_b), "fused records differ from UpdateDepth + RunStep"
    assert al.unpack(rec_b)[0].inliers > 0.3 * w * h


def test_sfm_evaluate_error_matches_oracle(torch_mod, oracle):
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner, SfmAlignerParams, DenseSfmParams
    pair = synth.make_pair(320, 240, 32, 1, seed=9, code_sigma=0.5)
    L = pair.levels[0]
    dev = upload_level(torch, L, 8)
    for delta in (0.1, 0.5):
        al = SfmAligner(32, SfmAlignerParams(sfmparams=DenseSfmParams(huber_delta=delta)))
        g = al.EvaluateError(pair.pose0, pair.pose1, L.cam, dev["img0"], dev["img1"], dev["dpt0"], dev["std0"],
                             dev["grad1"])
        res, inl = oracle.sfm_evaluate_error(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0,
                                             oracle.default_params(huber_delta=delta), precision="f64")
        assert g.inliers == inl
        assert abs(g.residual - res) <= 1e-5 * res


def test_se3_run_step_and_warp_match_oracle(torch_mod, oracle, golden):
    torch = torch_mod
    from deepfactors_b200.aligners import SE3Aligner
    from helpers import scenenet_inputs
    cam, img0, img1, dpt0 = scenenet_inputs(golden)
    grad1 = oracle.sobel_gradients(img1)
    d = dict(img0=pitched(torch, img0, 4), img1=pitched(torch, img1), dpt0=pitched(torch, dpt0),
             grad1=pitched(torch, grad1))
    al = SE3Aligner()
    for pose in (se3.identity(), se3.make_pose([0.01, -0.02, 0.005], [0.02, 0.01, -0.01])):
        g = al.RunStep(pose, cam, d["img0"], d["img1"], d["dpt0"], d["grad1"])
        o32 = oracle.se3_run_step(pose, cam, img0, img1, dpt0, grad1, 0.1, precision="f32")
        o64 = oracle.se3_run_step(pose, cam, img0, img1, dpt0, grad1, 0.1, precision="f64")
        assert g.inliers == o32.inliers  # bit-identical validity chain (fp32 CPU path)
        # the fp64 truth can disagree with fp32 on pixels sitting exactly on the border (identity pose)
        ref, k = (o64, 1.0) if o64.inliers == o32.inliers else (o32, 2.0)
        assert np.abs(g.JtJ - ref.JtJ).max() <= k * H_TOL * np.abs(ref.JtJ).max()
        assert np.abs(g.Jtr - ref.Jtr).max() <= k * JTR_TOL * np.abs(ref.Jtr).max()
        assert abs(g.residual - ref.residual) <= k * RES_TOL * ref.residual
        img2 = torch.full((240, 320), -1.0, device="cuda")
        w = al.Warp(pose, cam, d["img0"], d["img1"], d["dpt0"], img2)
        img2_cpu, res, inl = oracle.se3_warp(pose, cam, img0, img1, dpt0, precision="f32")
        assert w.inliers == inl
        assert abs(w.residual - res) <= 1e-3 * max(1.0, abs(res))
        assert np.abs(img2.cpu().numpy() - img2_cpu).max() <= 1e-6


def test_se3_image_alignment_converges_on_gpu(torch_mod, oracle, golden):
    """tests/ut_se3aligner.cpp:173-211 run through the CUDA path: 40 GN iterations, error <= 1e-3"""
    torch = torch_mod
    from deepfactors_b200.aligners import SE3Aligner, SobelGradients
    from helpers import scenenet_inputs
    cam, img0, img1, dpt0 = scenenet_inputs(golden)
    d0, d1, dd = pitched(torch, img0), pitched(torch, img1), pitched(torch, dpt0)
    grad = torch.zeros((240, 320, 2), device="cuda")
    SobelGradients(d1, grad)
    al = SE3Aligner()
    pose = se3.identity(np.float64)
    err = None
    for _ in range(40):
        r = al.RunStep(pose.astype(np.float32), cam, d0, d1, dd, grad)
        pose = se3.se3_solve_and_update(r.toDenseMatrix(), r.Jtr, pose)
        err = r.residual / r.inliers
    assert err <= 1e-3


def test_camera_tracker_device_loop_matches_host_loop(torch_mod, oracle, golden):
    """CameraTracker::TrackFrame (camera_tracker.cpp:42-69) with the whole coarse-to-fine loop on the device:
    every iteration's system == the oracle's at the same pose, every on-device LDLT + retraction == numpy's,
    the final pose / inlier fraction / error == the oracle's host loop."""
    torch = torch_mod
    from deepfactors_b200.aligners import CameraTracker, TrackerConfig
    from helpers import tracking_pyramid
    cams, p0, p1, pd, pg = tracking_pyramid(golden, oracle, 3)
    iters = (10, 5, 4)
    cfg = TrackerConfig(pyramid_levels=3, iterations_per_level=iters, huber_delta=0.1)
    trk = CameraTracker(cams, cfg)
    up = lambda lst, extra=0: [pitched(torch, a, extra) for a in lst]
    trk.SetKeyframe(up(p0), up(pd, 3))
    pose = trk.TrackFrame(up(p1, 5), up(pg), keep_history=True)
    o_pose, o_frac, o_err, o_hist = oracle.se3_track(se3.identity(np.float64), cams, p0, p1, pd, pg, iters, 0.1)
    hist = trk.history_
    assert hist.shape == (sum(iters), 36) and len(o_hist) == sum(iters)
    # first iteration: same pose (identity) -> the strict single-step bar
    # (identity pose: pixels sit exactly on the validity border, so the fp32 CPU flavour is the comparable one)
    g0 = hist[0]
    r0 = oracle.se3_run_step(se3.identity(), cams[2], p0[2], p1[2], pd[2], pg[2], 0.1)
    assert int(g0[28:29].view(np.uint32)[0]) == r0.inliers
    assert np.abs(g0[:21] - r0.JtJ).max() <= 4e-5 * np.abs(r0.JtJ).max()
    # every iteration: the pose of iteration k+1 is numpy's solve + retraction applied to the device's own system k
    level_of = [l for l in (2, 1, 0) for _ in range(iters[l])]
    for k in range(len(hist) - 1):
        Hk = np.zeros((6, 6))
        Hk[np.triu_indices(6)] = hist[k][:21].astype(np.float64)
        Hk = Hk + np.triu(Hk, 1).T
        want = se3.se3_solve_and_update(Hk, hist[k][21:27].astype(np.float64), hist[k][29:36].astype(np.float64))
        assert np.abs(want - hist[k + 1][29:36]).max() <= 5e-6, f"on-device update of iteration {k}"
        # and the device's system at its pose == the CPU path's at that same pose: inliers exactly (the fp32 flavour, as
        # in ut_sfmaligner.cpp:320 -- at 80x60 a single border pixel that flips between fp32 and fp64 is 2e-4 of the sum)
        lv = level_of[k]
        r32 = oracle.se3_run_step(hist[k][29:36], cams[lv], p0[lv], p1[lv], pd[lv], pg[lv], 0.1, precision="f32")
        assert int(hist[k][28:29].view(np.uint32)[0]) == r32.inliers, f"inliers of iteration {k}"
        assert np.abs(hist[k][:21] - r32.JtJ).max() <= 1e-4 * np.abs(r32.JtJ).max(), f"system of iteration {k}"
    # end result vs the oracle's own loop (fp64 steps, numpy solve)
    assert np.abs(pose - o_pose).max() <= 2e-4, (pose, o_pose)
    assert abs(trk.GetInliers() - o_frac) <= 2e-3
    assert abs(trk.GetError() - o_err) <= 1e-3 * o_err
    # a second frame continues from the tracked pose (camera_tracker.cpp keeps pose_ck_ across frames)
    before = trk.GetError()
    trk.TrackFrame(up(p1), up(pg))
    assert trk.GetError() <= before * 1.0001


def test_camera_tracker_converges_and_handles_no_overlap(torch_mod, oracle, golden):
    """tests/ut_se3aligner.cpp:173-211 as one device-side loop: 40 GN iterations at level 0, error <= 1e-3; and a pose
    with zero overlap leaves the estimate untouched with error = +inf (camera_tracker.cpp:68)"""
    torch = torch_mod
    from deepfactors_b200.aligners import CameraTracker, TrackerConfig
    from helpers import tracking_pyramid
    cams, p0, p1, pd, pg = tracking_pyramid(golden, oracle, 1)
    trk = CameraTracker(cams, TrackerConfig(pyramid_levels=1, iterations_per_level=(40,), huber_delta=0.1))
    up = lambda lst: [pitched(torch, a) for a in lst]
    trk.SetKeyframe(up(p0), up(pd))
    trk.TrackFrame(up(p1), up(pg))
    assert trk.GetError() <= 1e-3 and trk.GetInliers() > 0.5
    far = se3.make_pose([0, 0, 0], [0, 0, -100.0])  # every keyframe point lands behind the live camera
    trk.pose_ck_ = far.copy()
    out = trk.TrackFrame(up(p1), up(pg))
    assert np.array_equal(out, far) and trk.GetError() == float("inf") and trk.GetInliers() == 0.0


def test_image_proc_matches_oracle_and_opencv(torch_mod, oracle, golden):
    torch = torch_mod
    from deepfactors_b200.aligners import GaussianBlurDown, SobelGradients, SquaredError, UpdateDepth
    img = golden["gray_1047"].astype(np.float32) * np.float32(1 / 255.0)
    dimg = pitched(torch, img, 4)
    grad = torch.zeros((240, 320, 2), device="cuda")
    SobelGradients(dimg, grad)
    g = grad.cpu().numpy()
    assert np.array_equal(g, oracle.sobel_gradients(img))  # same operation order => bit exact
    assert np.abs(g[1:-1, 1:-1, 0] - golden["ocv_sobel_x_1047"][1:-1, 1:-1]).max() < 1e-4  # ut_cuda_utils.cpp:140
    down = torch.zeros((120, 160), device="cuda")
    GaussianBlurDown(dimg, down)
    dn = down.cpu().numpy()
    assert np.abs(dn - oracle.gaussian_blur_down(img)).max() <= 1e-7
    assert np.abs(dn[1:-1, 1:-1] - golden["ocv_blurdown_1047"][1:-1, 1:-1]).max() < 1e-1  # ut_cuda_utils.cpp:101
    other = pitched(torch, golden["gray_1052"].astype(np.float32) / 255.0)
    se = SquaredError(dimg, other)
    ref = oracle.squared_error(img, (golden["gray_1052"].astype(np.float32) / 255.0).astype(np.float32), "f64")
    assert abs(se - ref) <= 1e-5 * ref
    # UpdateDepth for every code size the ABI vectorises + one generic size
    rng = np.random.default_rng(0)
    for cs in (8, 32, 128, 12):
        prx = (0.5 + 0.4 * rng.random((60, 80))).astype(np.float32)
        jac = (rng.standard_normal((60, 80, cs)) * 0.02).astype(np.float32)
        code = (rng.standard_normal(cs) * (4.0 / np.sqrt(cs))).astype(np.float32)  # |jac.code| ~ 0.08 << prx
        out = torch.zeros((60, 80), device="cuda")
        UpdateDepth(code, pitched(torch, prx), pitched(torch, jac), 2.0, out)
        ref = oracle.update_depth(code, prx, jac, 2.0)
        assert np.all(np.abs(out.cpu().numpy() - ref) <= 1e-5 * np.abs(ref) + 1e-6)


def test_build_image_pyramid_matches_per_level_calls(torch_mod, oracle, golden):
    """Frame::FillPyramids (frame.h:80-94): blur-down chain + Sobel per level in one enqueue == the oracle's chain"""
    torch = torch_mod
    from deepfactors_b200.aligners import BuildImagePyramid
    img = golden["gray_1047"].astype(np.float32) * np.float32(1 / 255.0)
    levels = 4
    imgs = [pitched(torch, img, 3)] + [torch.zeros((240 >> l, 320 >> l), device="cuda") for l in range(1, levels)]
    grads = [torch.zeros((240 >> l, 320 >> l, 2), device="cuda") for l in range(levels)]
    BuildImagePyramid(imgs, grads)
    torch.cuda.synchronize()
    ref = img
    for l in range(levels):
        if l:
            ref = oracle.gaussian_blur_down(ref)
        assert np.abs(imgs[l].cpu().numpy() - ref).max() <= 1e-6
        g = oracle.sobel_gradients(imgs[l].cpu().numpy())
        assert np.array_equal(grads[l].cpu().numpy(), g)


def test_error_reporting_is_loud(torch_mod):
    torch = torch_mod
    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(32)
    pair = synth.make_pair(160, 120, 32, 1)
    L = pair.levels[0]
    dev = upload_level(torch, L)
    with pytest.raises((_lib.DfkError, ValueError)):  # mismatched view sizes
        al.RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"][:100], dev["img1"], dev["dpt0"], None,
                   dev["valid0"], dev["prx0_jac"], dev["grad1"])
    with pytest.raises(_lib.DfkError):  # threads must be a multiple of 32 (cu_sfmaligner.cpp:190)
        al.SetStepThreadsBlocks(33, 11)
    bad = SfmAligner(5)  # no kernel for this code size
    with pytest.raises((_lib.DfkError, ValueError)):
        bad.RunStep(pair.pose0, pair.pose1, None, L.cam, dev["img0"], dev["img1"], dev["dpt0"], None, dev["valid0"],
                    dev["prx0_jac"], dev["grad1"])


@pytest.mark.parametrize("cs", [8, 32])
def test_sfm_failed_batch_leaves_no_unbuilt_ray_table(torch_mod, cs):
    """a call that names a new camera level and then fails on a later item must not leave that level's ray table unbuilt
    in the handle's cache: the next call on the level equals a fresh handle's, bit for bit"""
    torch = torch_mod
    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner
    pair = synth.make_pair(160, 120, cs, 1, seed=71, code_sigma=0.5)
    L = pair.levels[0]
    dev = upload_level(torch, L)
    good = dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam,
                **{k: dev[k] for k in ("img0", "img1", "dpt0", "valid0", "prx0_jac", "grad1")})
    al = SfmAligner(cs)
    with pytest.raises(_lib.DfkError):  # img1 smaller than img0: rejected after the first item
        al.RunStepBatch(al.make_work_items([good, dict(good, img1=dev["img1"][:100])]))
    va, vb = torch.zeros_like(dev["valid0"]), torch.zeros_like(dev["valid0"])
    got = al.RunStepBatch(al.make_work_items([dict(good, valid0=va)])).clone()
    fresh = SfmAligner(cs)
    want = fresh.RunStepBatch(fresh.make_work_items([dict(good, valid0=vb)])).clone()
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert torch.equal(va, vb)


@pytest.mark.gpu
def test_window_assembly_on_device_matches_host_mirror():
    """dfk_window_assemble (deterministic gather over the record buffer of a batch) == factors.WindowBlocks.pack on the
    same records == the dense window of factors.assemble_window; 5 keyframes, 7 pairs x 2 levels, C = 32 and 8."""
    import torch
    from deepfactors_b200 import factors
    from deepfactors_b200.aligners import SfmAligner, Window
    for cs in (32, 8):
        n_kf = 5
        pairs = [(0, 1), (1, 2), (2, 3), (3, 4), (4, 0), (0, 2), (3, 1)]
        al = SfmAligner(cs)
        items, item_pair, sizes = [], [], []
        for p, (k0, k1) in enumerate(pairs):
            pr = synth.make_pair(160, 120, cs, 2, seed=40 + p, code_sigma=0.2, phase=0.05 * p)
            for L in pr.levels:
                d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
                    img0=L.img0, img1=L.img1, dpt0=L.dpt0, prx0_jac=L.prx_jac, grad1=L.grad1).items()}
                items.append(dict(pose0=pr.pose0, pose1=pr.pose1, cam=L.cam, valid0=torch.zeros_like(d["img0"]), **d))
                item_pair.append(p)
                sizes.append((L.width, L.height))
        work = al.make_work_items(items)
        recs = al.RunStepBatch(work)
        win = Window(al, n_kf, pairs, item_pair, sizes)
        buf = win.assemble(recs)
        buf2 = win.assemble(recs)
        torch.cuda.synchronize()
        assert torch.equal(buf, buf2)                                  # deterministic (a gather, no float atomics)
        H, g, res, inl = factors.unpack_records(recs.cpu().numpy(), cs)
        want = win.layout.pack(item_pair, H, g, res, inl, sizes)
        got = buf.cpu().numpy()
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= 2e-6 * np.abs(want).max()  # two fp32 summation orders of <= 6 terms
        Hd, gd, f, ninl = win.layout.to_dense(got)
        Hr, gr, fr = factors.assemble_window(factors.WindowLayout(n_kf, cs), [pairs[p] for p in item_pair], H, g, res, inl,
                                             sizes)
        assert np.abs(Hd - Hr).max() <= 2e-6 * np.abs(Hr).max() and np.abs(gd - gr).max() <= 2e-6 * np.abs(gr).max()
        assert abs(f - fr) <= 1e-5 * abs(fr) and ninl == float(inl.sum())
        assert np.allclose(Hd, Hd.T)


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,cs", [(160, 120, 32), (80, 60, 8), (97, 33, 16), (64, 48, 128)])
def test_depth_aligner_run_step_matches_oracle(oracle, w, h, cs):
    """DepthAligner::RunStep (cu_depthaligner.cpp:32-113) vs the CPU oracle (fp64): every pixel counts."""
    import torch
    from deepfactors_b200.aligners import DepthAligner
    L = synth.make_level(w, h, cs, seed=8)
    code = (np.random.default_rng(3).standard_normal(cs) * 0.3).astype(np.float32)
    tgt = (L.dpt0 * np.float32(1.05) + np.float32(0.02)).astype(np.float32)
    da = DepthAligner(cs)
    g = da.RunStep(code, pitched(torch, tgt, 3), pitched(torch, L.prx_orig), pitched(torch, L.prx_jac, 4))
    o = oracle.depth_run_step(code, tgt, L.prx_orig, L.prx_jac, 2.0, precision="f64")
    assert g.inliers == o.inliers == w * h
    assert np.abs(g.JtJ - o.JtJ).max() <= 2e-5 * np.abs(o.JtJ).max()
    assert np.abs(g.Jtr - o.Jtr).max() <= 1e-4 * np.abs(o.Jtr).max()
    assert abs(g.residual - o.residual) <= 1e-5 * abs(o.residual)
    g2 = da.RunStep(code, pitched(torch, tgt, 3), pitched(torch, L.prx_orig), pitched(torch, L.prx_jac, 4))
    assert np.array_equal(g.JtJ, g2.JtJ)  # fixed summation order


@pytest.mark.gpu
def test_streaming_from_host_matches_device_resident_batch():
    """dfk_sfm_stream_submit / _wait (host image views, pipelined upload) returns the records of the device-resident
    batch, bit for bit, for several submissions in flight."""
    import ctypes as C
    import torch
    from deepfactors_b200 import _lib
    from deepfactors_b200._lib import DfkCamera, DfkImage, DfkSfmWorkItem
    from deepfactors_b200.aligners import SfmAligner
    cs = 32
    al = SfmAligner(cs)
    lib = _lib.lib()
    rec = _lib.record_floats(cs)
    pairs = [synth.make_pair(160, 120, cs, 2, seed=60 + k, code_sigma=0.2) for k in range(4)]
    want = []
    for pr in pairs:
        items = []
        for L in pr.levels:
            d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
                img0=L.img0, img1=L.img1, dpt0=L.dpt0, prx0_jac=L.prx_jac, grad1=L.grad1).items()}
            items.append(dict(pose0=pr.pose0, pose1=pr.pose1, cam=L.cam, valid0=torch.zeros_like(d["img0"]), **d))
        want.append(al.RunStepBatch(al.make_work_items(items)).cpu().numpy())
    keep, arrs = [], []
    for pr in pairs:
        arr = (DfkSfmWorkItem * 2)()
        for l, L in enumerate(pr.levels):
            t = {k: torch.from_numpy(np.ascontiguousarray(v)).pin_memory() for k, v in dict(
                img0=L.img0, img1=L.img1, dpt0=L.dpt0, prx0_jac=L.prx_jac, grad1=L.grad1).items()}
            keep.append(t)
            w = arr[l]
            w.pose0 = (C.c_float * 7)(*np.asarray(pr.pose0, dtype=np.float32).tolist())
            w.pose1 = (C.c_float * 7)(*np.asarray(pr.pose1, dtype=np.float32).tolist())
            w.cam = DfkCamera(L.cam.fx, L.cam.fy, L.cam.u0, L.cam.v0, L.cam.width, L.cam.height)
            im = lambda x: DfkImage(C.c_void_p(x.data_ptr()), x.stride(0) * 4, x.shape[1], x.shape[0])
            w.img0, w.img1, w.dpt0, w.prx0_jac, w.grad1 = im(t["img0"]), im(t["img1"]), im(t["dpt0"]), im(t["prx0_jac"]), im(t["grad1"])
        arrs.append(arr)
    al._hd.use_torch_stream()
    st = C.c_void_p()
    _lib.check(al.handle, lib.dfk_sfm_stream_create(al.handle, cs, 2, 1 << 16, 3, C.byref(st)))  # small hint: slots must grow
    tk = C.c_uint64(0)
    for arr in arrs[:3]:
        _lib.check(al.handle, lib.dfk_sfm_stream_submit(al.handle, st, arr, 2, C.byref(tk)))
    # a fourth submission with three outstanding is refused, waiting out of order too
    assert lib.dfk_sfm_stream_submit(al.handle, st, arrs[3], 2, C.byref(tk)) == _lib.DFK_ERR_INVALID_ARG
    out = np.zeros((2, rec), dtype=np.float32)
    op = out.ctypes.data_as(C.POINTER(C.c_float))
    assert lib.dfk_sfm_stream_wait(al.handle, st, C.c_uint64(1), op) == _lib.DFK_ERR_INVALID_ARG
    for k in range(3):
        _lib.check(al.handle, lib.dfk_sfm_stream_wait(al.handle, st, C.c_uint64(k), op))
        assert np.array_equal(out, want[k]), f"submission {k}"
        if k == 0:
            _lib.check(al.handle, lib.dfk_sfm_stream_submit(al.handle, st, arrs[3], 2, C.byref(tk)))
    _lib.check(al.handle, lib.dfk_sfm_stream_wait(al.handle, st, C.c_uint64(3), op))
    assert np.array_equal(out, want[3])
    lib.dfk_sfm_stream_destroy(al.handle, st)


@pytest.mark.gpu
def test_window_gauss_newton_loop_on_device_recovers_perturbed_poses():
    """window_opt.SfmWindowProblem + WindowOptimizer: 3 keyframes that see the same scene from the same pose (so the truth
    is 'all relative poses identity, zero codes'), poses of keyframes 1 and 2 perturbed; LM over poses + codes with the
    linearisation in one batched fused-decode launch and the assembly on the device must bring the energy down by > 20x
    and the poses back towards identity.  First linearisation also checked against the host mirror of the assembly."""
    import torch
    from deepfactors_b200 import factors
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import LMParams, SfmWindowProblem, WindowOptimizer
    cs, levels = 8, 2
    base = synth.make_pair(160, 120, cs, levels, seed=5)
    cams = [L.cam for L in base.levels]
    al = SfmAligner(cs)
    keyframes = []
    for k in range(3):
        lv = []
        for L in base.levels:
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
            img = up(L.img0)
            lv.append(dict(img=img, grad=up(synth.sobel_np(L.img0)), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac),
                           dpt=torch.zeros_like(img), valid=torch.zeros_like(img)))
        keyframes.append(lv)
    pairs = [(0, 1), (1, 2), (2, 0), (1, 0), (2, 1)]
    prob = SfmWindowProblem(al, cams, keyframes, pairs)
    poses = np.stack([se3.identity(np.float64),
                      se3.make_pose([0.004, -0.003, 0.002], [0.015, -0.01, 0.008], np.float64),
                      se3.make_pose([-0.003, 0.002, 0.004], [-0.01, 0.012, -0.006], np.float64)])
    codes = np.zeros((3, cs))
    # one linearisation by hand: device assembly == host mirror on the same records
    buf, _ = prob.linearise(poses, codes, list(range(len(pairs))))
    torch.cuda.synchronize()
    H, g, res, inl = factors.unpack_records(prob.records.cpu().numpy(), cs)
    item_pair = [p for p in range(len(pairs)) for _ in range(levels)]
    sizes = [(L.width, L.height) for _ in pairs for L in base.levels]
    want = prob.layout.pack(item_pair, H, g, res, inl, sizes)
    assert np.abs(buf.cpu().numpy() - want).max() <= 2e-6 * np.abs(want).max()
    opt = WindowOptimizer(prob.layout, prob.linearise, LMParams(iterations=12, lambda_init=1e-3, code_prior_weight=1e-2))
    p, c, tr = opt.run(poses, codes)
    assert tr.energy[-1] < tr.energy[0] / 20.0, tr.energy
    err0 = max(np.abs(poses[k][4:7]).max() for k in (1, 2))
    err1 = max(np.abs(p[k][4:7] - p[0][4:7]).max() for k in (1, 2))
    assert err1 < 0.25 * err0, (err0, err1)
    assert np.allclose(p[0], poses[0])                      # gauge keyframe fixed
    assert tr.factors_relinearised[0] == len(pairs)


@pytest.mark.gpu
@pytest.mark.parametrize("cs", [32, 8])
def test_reprojection_factor_rows_on_device_match_oracle(oracle, cs):
    """dfk_reprojection_linearize (rows gathered on the device, reprojection_factor.cpp:157-269) vs the CPU oracle"""
    import torch
    from deepfactors_b200.aligners import ReprojectionLinearize, SfmAligner
    from test_oracle_ref import _keypoint_matches
    L = synth.make_level(160, 120, cs, seed=12)
    pose0, pose1 = synth.reference_test_poses()
    code = (np.random.default_rng(5).standard_normal(cs) * 0.3).astype(np.float32)
    q, t = _keypoint_matches(L.cam, pose0, pose1, L.prx_orig, n=1000)
    q[3] = [-4.0, 7.0]     # outside the image: zero rows instead of the reference's out-of-bounds read
    al = SfmAligner(cs)
    rows, tot = ReprojectionLinearize(al, pose0, pose1, code, L.cam, pitched(torch, L.prx_orig, 3), pitched(torch, L.prx_jac, 2),
                                      q, t, 1.5, 2.0)
    r64, e64 = oracle.reprojection_rows(pose0, pose1, code, L.cam, L.prx_orig, L.prx_jac, q, t, 1.5, 2.0, precision="f64")
    assert rows.shape == r64.shape and not rows[6:8].any()
    assert np.abs(rows - r64).max() <= 1e-4 * np.abs(r64).max()
    assert abs(tot - e64) <= 1e-4 * e64


@pytest.mark.gpu
@pytest.mark.parametrize("cs", [32, 8])
def test_sparse_geometric_factor_rows_on_device_match_oracle(oracle, cs):
    """dfk_sparse_geometric_linearize (sparse_geometric_factor.cpp:157-271 on the device) vs the CPU oracle: the same set
    of valid rows (exact-order decode + validity chain), every block of the rows within fp32 rounding of the fp64 oracle"""
    import torch
    from deepfactors_b200.aligners import SfmAligner, SparseGeometricLinearize
    from test_oracle_ref import _geometric_scene
    L0, L1, code0, code1, g1, pts = _geometric_scene(cs)
    pts = np.concatenate([pts, np.array([[-3, 5], [200, 10]], dtype=np.int32)])   # outside the image: zero rows
    pose0, pose1 = synth.reference_test_poses()
    al = SfmAligner(cs)
    rows, nv = SparseGeometricLinearize(al, pose0, pose1, code0, code1, L0.cam, pitched(torch, L0.prx_orig, 3),
                                        pitched(torch, L0.prx_jac, 2), pitched(torch, L1.prx_orig, 1),
                                        pitched(torch, L1.prx_jac, 4), pitched(torch, g1, 2), pts, 0.1)
    args = (pose0, pose1, code0, code1, L0.cam, L0.prx_orig, L0.prx_jac, L1.prx_orig, L1.prx_jac, g1, pts, 0.1)
    r32, n32 = oracle.sparse_geometric_rows(*args)
    r64, n64 = oracle.sparse_geometric_rows(*args, precision="f64")
    assert rows.shape == r64.shape and not rows[-2:].any()
    assert nv == n32 and 0 < nv < pts.shape[0]
    assert np.array_equal(np.abs(rows).sum(1) > 0, np.abs(r32).sum(1) > 0), "valid set differs from the fp32 CPU path"
    same = (np.abs(r64).sum(1) > 0) == (np.abs(r32).sum(1) > 0)   # fp64 may disagree on a point that sits on the border
    for sl in (slice(0, 6), slice(6, 12), slice(12, 12 + cs), slice(12 + cs, 12 + 2 * cs), slice(12 + 2 * cs, None)):
        assert np.abs(rows[same][:, sl] - r64[same][:, sl]).max() <= 2e-4 * np.abs(r64[:, sl]).max()
    # loud errors
    with pytest.raises(Exception):
        SparseGeometricLinearize(al, pose0, pose1, code0, code1, L0.cam, pitched(torch, L0.prx_orig, 3),
                                 pitched(torch, L0.prx_jac, 2), pitched(torch, L1.prx_orig[:-2], 1),
                                 pitched(torch, L1.prx_jac, 4), pitched(torch, g1, 2), pts, 0.1)
