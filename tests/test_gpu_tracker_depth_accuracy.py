"""The tracker's SE3 step, the thin reductions around it, DepthAligner and UpdateDepth against fp64, entry by entry, at
the sizes where their grid-stride loops and block caps engage (system_accuracy.py has the scales and the bars).

The SE3 kernels run a grid of at most 1024 blocks x 256 threads = 262 144 threads; 320x240 needs 300 blocks, so until
now every thread handled one pixel.  Here 640x480 (1200 blocks' worth, capped) and 1280x960 (4.7 pixels per thread)
take the second and later grid-stride passes and finalize 1024 partials.

Covered, each case printing its worst entry (block, index, ratio to its scale):
  * SE3Aligner::RunStep at 80x60, 320x240, 640x480, 1280x960, 33x7 and 5x5; dense, pitched, and a grad1 view one float
    off 8-byte alignment (the unaligned gradient path); Huber delta 0.01, 0.1 and 10 through SetHuberDelta.  Every
    entry of JtJ within 5e-5 S, of Jtr within 1e-6 B (1e-5 B below 64 valid pixels: one pixel's front-end rounding
    does not average out, test_gpu_system_accuracy.py has the analysis), residual 1e-5, inliers exact.  The fp64 rows
    take their pixel set from the fp32 validity chain.
  * CameraTracker on a 4-level 640x480 pyramid with keep_history: the 29-float system of every iteration against fp64
    at the pose the device evaluated it at, Jtr included, started near the minimum; the last iterations are asserted
    to be in the cancellation regime (max |Jtr| << max B).
  * TrackFrameBatch at 640x480 and 1280x960 with mixed sizes: bit for bit what single dfk_se3_track gives.
  * Zero overlap from a rotated start, single and batched: the pose comes back bit for bit, error +inf.
  * EvaluateError, Warp, SquaredError at the same sizes (SquaredError also 1x1): inliers equal to the fp32 oracle,
    EvaluateError / SquaredError residuals within 1e-5 / 1e-6 relative of fp64, Warp's signed residual within
    1e-6 sum |img0 - sampled| of fp64, the warped image and pitched outputs.
  * DepthAligner at C = 8 .. 128 up to 1280x960, areas that are not a multiple of 64, pitched views, zero-mean and
    one-signed Jacobian columns, avg_dpt != 2 through the aligner params.
  * UpdateDepth on every dispatch path: C = 4 .. 128 vectorised, the same C with a misaligned Jacobian view (generic
    kernel), C = 1, 3, 12, 256; 1x1 to 1280x960 with pitched output; every pixel within 1e-6 S_px of fp64.
  * SobelGradients / GaussianBlurDown bit-exact against the oracle on partial 32x8 blocks (1x1, 1x37, 37x1, 33x9,
    31x7) with pitched input and output, blur-down from 81x61 and 3x3, and BuildImagePyramid from 1282x962.
"""
import numpy as np
import pytest

from deepfactors_b200 import se3, synth
from system_accuracy import (CODE_NAMES, JTR_BAR, SE3_NAMES, UD_BAR, assert_system_close, depth_reference,
                             se3_reference, update_depth_errors, update_depth_scale)

pytestmark = pytest.mark.gpu

POSE = se3.make_pose([0.01, -0.02, 0.005], [0.02, 0.01, -0.03])
SE3_SIZES = [(80, 60), (320, 240), (640, 480), (1280, 960), (33, 7), (5, 5)]


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def upload(torch, arr, extra_px=0, offset=0):
    """host [H, W(, K)] -> device view whose rows are padded by extra_px pixels and which starts `offset` floats into
    its buffer; the padding is NaN, so a read outside the view shows in the result"""
    a = np.ascontiguousarray(arr, dtype=np.float32)
    h, w = a.shape[:2]
    k = a.shape[2] if a.ndim == 3 else 1
    row = (w + extra_px) * k
    buf = torch.full((h * row + offset + 4,), float("nan"), dtype=torch.float32, device="cuda")
    flat = torch.as_strided(buf, (h, w * k), (row, 1), offset)
    flat.copy_(torch.from_numpy(a.reshape(h, w * k)))
    return flat if a.ndim == 2 else torch.as_strided(buf, (h, w, k), (row, k, 1), offset)


def output(torch, h, w, k=1, extra_px=0):
    """an output view with NaN padding (checked with untouched_padding afterwards)"""
    return upload(torch, np.full((h, w, k) if k > 1 else (h, w), np.nan, np.float32), extra_px)


def untouched_padding(view, w, k=1):
    import torch
    row = view.stride(0)
    h = view.shape[0]
    buf = torch.as_strided(view, (h, row), (row, 1))
    return bool(torch.isnan(buf[:, w * k:]).all()) if row > w * k else True


def _small_jtr_bar(n):
    return JTR_BAR if n >= 64 else 1e-5


# ---------------------------------------------------------------------------------------------- SE3 RunStep
@pytest.mark.parametrize("w,h", SE3_SIZES)
@pytest.mark.parametrize("layout", ["dense", "pitched", "grad_unaligned"])
def test_se3_run_step_per_entry(torch_mod, w, h, layout):
    from deepfactors_b200.aligners import SE3Aligner
    torch = torch_mod
    L = synth.make_level(w, h, 1, seed=w + h)
    extra = 0 if layout == "dense" else 3
    d = {k: upload(torch, getattr(L, k), extra) for k in ("img0", "img1", "dpt0")}
    d["grad1"] = upload(torch, L.grad1, extra, offset=1 if layout == "grad_unaligned" else 0)
    al = SE3Aligner()
    for delta in (0.01, 0.1, 10.0):
        al.SetHuberDelta(delta)
        got = al.RunStep(POSE, L.cam, d["img0"], d["img1"], d["dpt0"], d["grad1"])
        ref = se3_reference(POSE, L.cam, L.img0, L.img1, L.dpt0, L.grad1, delta)
        what = f"SE3 {w}x{h} {layout} delta={delta} ({ref.inliers} px)"
        if ref.inliers == 0:
            assert got.inliers == 0 and not np.any(got.JtJ) and not np.any(got.Jtr) and got.residual == 0.0, what
            continue
        assert_system_close(got, ref, ref.S, ref.B, what, jtr_bar=_small_jtr_bar(ref.inliers), names=SE3_NAMES)
    if w * h >= 320 * 240:
        assert ref.inliers > 0.5 * w * h


# ---------------------------------------------------------------------------------------------- tracker
def tracking_pyramid(w=640, h=480, levels=4, seed=11, extra_px=0):
    """keyframe image / depth and a live frame whose photometric minimum is near the identity: img1 = img0 plus a small
    independent texture, so the minimum keeps a residual and Jtr cancels there"""
    pair = synth.make_pair(w, h, 1, levels, seed=seed, identity_pose=True)
    cams, p0, pd, p1, pg = [], [], [], [], []
    for L in pair.levels:
        img1 = (L.img0 + np.float32(0.05) * (L.img1 - np.float32(0.5))).astype(np.float32)
        cams.append(L.cam)
        p0.append(L.img0)
        pd.append(L.dpt0)
        p1.append(img1)
        pg.append(synth.sobel_np(img1))
    return cams, p0, pd, p1, pg


def test_tracker_iterations_per_entry(torch_mod):
    from deepfactors_b200.aligners import CameraTracker, JTJJrReductionItem, TrackerConfig
    torch = torch_mod
    cams, p0, pd, p1, pg = tracking_pyramid()
    iters = (4, 4, 4, 4)
    tr = CameraTracker(cams, TrackerConfig(4, iters, 0.1))
    tr.SetKeyframe([upload(torch, a) for a in p0], [upload(torch, a) for a in pd])
    tr.pose_ck_ = se3.make_pose([0.004, -0.003, 0.002], [0.01, -0.008, 0.005])
    tr.TrackFrame([upload(torch, a) for a in p1], [upload(torch, a) for a in pg], keep_history=True)
    hist = tr.history_
    level_of = [l for l in range(3, -1, -1) for _ in range(iters[l])]
    last_ratio = None
    for k, (row, l) in enumerate(zip(hist, level_of)):
        pose = row[29:36].copy()
        got = JTJJrReductionItem(row[:21].copy(), row[21:27].copy(), float(row[27]),
                                 int(np.ascontiguousarray(row[28:29]).view(np.uint32)[0]))
        ref = se3_reference(pose, cams[l], p0[l], p1[l], pd[l], pg[l], 0.1)
        cancel = float(np.abs(ref.Jtr).max() / ref.B.max())
        assert_system_close(got, ref, ref.S, ref.B, f"tracker iteration {k} level {l} (max|Jtr|/max B {cancel:.1e})",
                            names=SE3_NAMES)
        if l == 0:
            last_ratio = cancel
    # the last level-0 iterations sum a Jtr that cancels: the GN step is driven by what a max-relative bar cannot see
    assert last_ratio < 1e-2, last_ratio
    assert tr.GetError() < np.inf


# ---------------------------------------------------------------------------------------------- track batch
def _problem(torch, w, h, pose, extra_px=0, seed=11, iters=(3, 3, 3, 3)):
    from test_gpu_track_batch import Problem
    cams, p0, pd, p1, pg = tracking_pyramid(w, h, 4, seed)
    return Problem(torch, cams, p0, pd, p1, pg, pose, extra_px=extra_px, iters=iters)


# every point behind the camera; the rotation is one whose fp32 quaternion is not a fixed point of an fp32
# renormalisation (q / |q| changes it whatever the order of the sum of squares, as for about 1 in 8 random rotations),
# so an update that renormalises without moving the pose still shows
FAR_ROTATED = se3.make_pose([-0.04, 0.32, 0.22], [0.0, 0.0, -100.0])


def test_track_batch_bit_for_bit_at_the_block_cap(torch_mod):
    """640x480 (1200 blocks' worth) and 1280x960 (4800) are capped at 1024 blocks per problem; mixed with smaller
    problems and a zero-overlap one in one batch, every problem still gives what dfk_se3_track gives alone"""
    from test_gpu_track_batch import assert_same, handle, track_batch, track_single
    torch = torch_mod
    start = se3.make_pose([0.004, -0.003, 0.002], [0.01, -0.008, 0.005])
    probs = {"640x480": _problem(torch, 640, 480, start),
             "1280x960": _problem(torch, 1280, 960, start, seed=12),
             "96x72": _problem(torch, 96, 72, start, seed=13),
             "640x480 pitched": _problem(torch, 640, 480, se3.identity(), extra_px=5, seed=14),
             "far rotated": _problem(torch, 320, 240, FAR_ROTATED, seed=15)}
    names = list(probs)
    singles = {k: track_single(p) for k, p in probs.items()}
    out = track_batch(handle(), [probs[k] for k in names])
    for n, k in enumerate(names):
        assert_same(out, n, singles[k], k)
        print(f"track batch {k}: pose {out[0][n]}, error {out[2][n]:.6e}, inliers {out[1][n]:.3f}")
    big = names.index("1280x960")
    assert np.isfinite(out[2][big]) and out[1][big] > 0.5


def test_zero_overlap_from_a_rotated_start_leaves_the_pose_alone(torch_mod):
    """no pixel is valid at any iteration: the pose must come back bit for bit (the reference skips the update when
    there are no inliers), error +inf, inlier fraction 0 -- single and batched"""
    from test_gpu_track_batch import bits, handle, track_batch, track_single
    torch = torch_mod
    prob = _problem(torch, 320, 240, FAR_ROTATED)
    pose, frac, err, sys_ = track_single(prob)
    print(f"zero overlap single: start {prob.pose} -> {pose}, error {err}")
    assert np.array_equal(bits(pose), bits(prob.pose)), (pose, prob.pose)
    assert err == np.inf and frac == 0.0 and bits(sys_[28]) == 0
    other = _problem(torch, 160, 120, se3.make_pose([0.004, -0.003, 0.002], [0.01, -0.008, 0.005]), seed=16)
    poses, fracs, errs, _ = track_batch(handle(), [other, prob, prob])
    for n in (1, 2):
        assert np.array_equal(bits(poses[n]), bits(prob.pose)), (poses[n], prob.pose)
        assert errs[n] == np.inf and fracs[n] == 0.0
    assert errs[0] < np.inf


# ---------------------------------------------------------------------------------------------- EvaluateError, Warp, SquaredError
@pytest.mark.parametrize("w,h", SE3_SIZES)
def test_evaluate_error_warp_per_size(torch_mod, w, h):
    from oracle import oracle as orc
    from deepfactors_b200.aligners import SE3Aligner, SfmAligner
    torch = torch_mod
    L = synth.make_level(w, h, 1, seed=w * 3 + h)
    d = {k: upload(torch, getattr(L, k), 2) for k in ("img0", "img1", "dpt0")}
    d["grad1"] = upload(torch, L.grad1, 2)
    ident = se3.identity()
    # EvaluateError: pose10 = pose1^-1 pose0 = POSE
    pose1 = se3.inverse(POSE.astype(np.float64), np.float32)
    ev = SfmAligner(8).EvaluateError(ident, pose1, L.cam, d["img0"], d["img1"], d["dpt0"], None, d["grad1"])
    r32, n32 = orc.sfm_evaluate_error(ident, pose1, L.cam, L.img0, L.img1, L.dpt0)
    r64, _ = orc.sfm_evaluate_error(ident, pose1, L.cam, L.img0, L.img1, L.dpt0, precision="f64")
    rel = abs(ev.residual - r64) / r64 if r64 else abs(ev.residual)
    print(f"EvaluateError {w}x{h}: inliers {ev.inliers} (fp32 oracle {n32}), residual {rel:.2e} relative (bar 1e-5)")
    assert ev.inliers == n32 and rel <= 1e-5
    # Warp: signed residual against fp64, scaled by sum |img0 - sampled|
    img2 = output(torch, h, w, extra_px=3)
    wp = SE3Aligner().Warp(POSE, L.cam, d["img0"], d["img1"], d["dpt0"], img2)
    i32, _, m32 = orc.se3_warp(POSE, L.cam, L.img0, L.img1, L.dpt0)
    i64, s64, _ = orc.se3_warp(POSE, L.cam, L.img0, L.img1, L.dpt0, precision="f64")
    scale = float(np.abs(L.img0.astype(np.float64) - i64)[i32 != 0].sum())
    ratio = abs(wp.residual - s64) / scale if scale else abs(wp.residual)
    print(f"Warp {w}x{h}: inliers {wp.inliers} (fp32 oracle {m32}), signed residual {ratio:.2e} of sum|diff| (bar 1e-6)")
    assert wp.inliers == m32 and ratio <= 1e-6
    got2 = img2.cpu().numpy()
    assert np.abs(got2 - i32).max() <= 1e-6 and untouched_padding(img2, w)


@pytest.mark.parametrize("w,h", SE3_SIZES + [(1, 1)])
def test_squared_error_per_size(torch_mod, w, h):
    from oracle import oracle as orc
    from deepfactors_b200.aligners import SquaredError
    rng = np.random.default_rng(w + h)
    a = rng.random((h, w), dtype=np.float32)
    b = rng.random((h, w), dtype=np.float32)
    got = SquaredError(upload(torch_mod, a, 3), upload(torch_mod, b, 1))
    ref = orc.squared_error(a, b, "f64")
    rel = abs(got - ref) / ref
    print(f"SquaredError {w}x{h}: {rel:.2e} relative (bar 1e-6)")
    assert rel <= 1e-6


# ---------------------------------------------------------------------------------------------- DepthAligner
DEPTH_CASES = [  # C, w, h, Jacobian columns, avg_dpt, row padding
    (8, 1280, 960, "one-signed", 2.0, 0), (16, 1280, 960, "zero-mean", 2.0, 3), (32, 1280, 960, "one-signed", 2.0, 0),
    (32, 640, 480, "zero-mean", 3.0, 4), (64, 321, 241, "zero-mean", 2.0, 3), (64, 640, 480, "one-signed", 1.5, 0),
    (128, 640, 480, "one-signed", 2.0, 0), (128, 97, 33, "zero-mean", 0.5, 1), (8, 37, 5, "one-signed", 2.0, 2),
]


def depth_case(cs, w, h, cols, avg):
    rng = np.random.default_rng(cs * 7 + w)
    L = synth.make_level(w, h, 1, seed=cs)
    jac = rng.standard_normal((h, w, cs)).astype(np.float32) * np.float32(0.02)
    if cols == "one-signed":
        jac = np.abs(jac)
    code = (rng.standard_normal(cs) * 0.3).astype(np.float32)
    if cols == "one-signed":
        code = np.abs(code)
    from oracle import oracle as orc
    dpt = orc.update_depth(code, L.prx_orig, jac, avg)
    if cols == "one-signed":  # the target one-signedly behind the decoded depth: nothing in Jtr cancels
        tgt = (dpt * np.float32(1.1)).astype(np.float32)
    else:
        tgt = (dpt + np.float32(0.05) * rng.standard_normal((h, w)).astype(np.float32)).astype(np.float32)
    return code, tgt, L.prx_orig, jac


@pytest.mark.parametrize("cs,w,h,cols,avg,extra", DEPTH_CASES)
def test_depth_aligner_per_entry(torch_mod, cs, w, h, cols, avg, extra):
    from deepfactors_b200.aligners import DenseSfmParams, DepthAligner, SfmAlignerParams
    torch = torch_mod
    code, tgt, prx, jac = depth_case(cs, w, h, cols, avg)
    al = DepthAligner(cs, params=SfmAlignerParams(sfmparams=DenseSfmParams(avg_dpt=avg)))
    got = al.RunStep(code, upload(torch, tgt, extra), upload(torch, prx, extra), upload(torch, jac, extra))
    ref = depth_reference(code, tgt, prx, jac, avg)
    assert_system_close(got, ref, ref.S, ref.B, f"DepthAligner C={cs} {w}x{h}+{extra} {cols} avg={avg}",
                        names=CODE_NAMES)


# ---------------------------------------------------------------------------------------------- UpdateDepth
def _ud_sizes(cs):
    if cs <= 32:
        return [(1, 1), (33, 7), (160, 120), (1280, 960)]
    if cs <= 128:
        return [(1, 1), (33, 7), (640, 480)]
    return [(1, 1), (33, 7), (160, 120)]


UD_CASES = ([(c, "aligned") for c in (4, 8, 16, 32, 64, 128)] + [(c, "misaligned") for c in (4, 16, 64, 128)] +
            [(c, "generic") for c in (1, 3, 12, 256)])


@pytest.mark.parametrize("cs,path", UD_CASES)
def test_update_depth_every_pixel(torch_mod, cs, path):
    from oracle import oracle as orc
    from deepfactors_b200.aligners import UpdateDepth
    torch = torch_mod
    for w, h in _ud_sizes(cs):
        rng = np.random.default_rng(cs + w)
        L = synth.make_level(w, h, 1, seed=cs)
        jac = (rng.standard_normal((h, w, cs)) * 0.02).astype(np.float32)
        code = (rng.standard_normal(cs) * 0.5).astype(np.float32)
        avg = 2.0 if w != 33 else 1.25
        jd = upload(torch, jac, 2 if w > 1 else 0, offset=1 if path == "misaligned" else 0)
        if cs == 1:  # a one-float-per-pixel Jacobian is a scalar image [H, W]
            jd = jd[:, :, 0]
        out = output(torch, h, w, extra_px=5)
        UpdateDepth(code, upload(torch, L.prx_orig, 1), jd, avg, out)
        got = out.cpu().numpy()
        ref = orc.update_depth(code, L.prx_orig, jac, avg, precision="f64")
        r, at = update_depth_errors(got, ref, update_depth_scale(code, L.prx_orig, jac, avg))
        print(f"UpdateDepth C={cs} {path} {w}x{h}: worst pixel {at} at {r:.2e} S_px (bar {UD_BAR:.0e})")
        assert r <= UD_BAR and untouched_padding(out, w)


# ---------------------------------------------------------------------------------------------- Sobel / blur-down
PARTIAL = [(1, 1), (1, 37), (37, 1), (33, 9), (31, 7)]


@pytest.mark.parametrize("w,h", PARTIAL)
def test_sobel_partial_blocks_bit_exact(torch_mod, w, h):
    from oracle import oracle as orc
    from deepfactors_b200.aligners import SobelGradients
    img = np.random.default_rng(w * 100 + h).random((h, w), dtype=np.float32)
    g = output(torch_mod, h, w, 2, extra_px=3)
    SobelGradients(upload(torch_mod, img, 2), g)
    assert np.array_equal(g.cpu().numpy(), orc.sobel_gradients(img)) and untouched_padding(g, w, 2), f"{w}x{h}"


@pytest.mark.parametrize("w,h", [(33, 9), (31, 7), (81, 61), (3, 3), (37, 2)])
def test_blur_down_odd_sizes_bit_exact(torch_mod, w, h):
    from oracle import oracle as orc
    from deepfactors_b200.aligners import GaussianBlurDown
    img = np.random.default_rng(w * 100 + h).random((h, w), dtype=np.float32)
    out = output(torch_mod, h // 2, w // 2, extra_px=3)
    GaussianBlurDown(upload(torch_mod, img, 2), out)
    assert np.array_equal(out.cpu().numpy(), orc.gaussian_blur_down(img)) and untouched_padding(out, w // 2), f"{w}x{h}"


def test_build_image_pyramid_from_1282x962_bit_exact(torch_mod):
    from oracle import oracle as orc
    from deepfactors_b200.aligners import BuildImagePyramid
    img = np.random.default_rng(5).random((962, 1282), dtype=np.float32)
    shapes = [(962, 1282)]
    for _ in range(3):
        shapes.append((shapes[-1][0] // 2, shapes[-1][1] // 2))
    imgs = [upload(torch_mod, img, 2)] + [output(torch_mod, h, w, extra_px=2) for h, w in shapes[1:]]
    grads = [output(torch_mod, h, w, 2, extra_px=1) for h, w in shapes]
    BuildImagePyramid(imgs, grads)
    ref = img
    for l, (h, w) in enumerate(shapes):
        if l:
            ref = orc.gaussian_blur_down(ref)
            assert np.array_equal(imgs[l].cpu().numpy(), ref), f"level {l} image"
        assert np.array_equal(grads[l].cpu().numpy(), orc.sobel_gradients(ref)), f"level {l} gradient"
        assert untouched_padding(grads[l], w, 2) and (l == 0 or untouched_padding(imgs[l], w))
