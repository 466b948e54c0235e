"""dfk_se3_track_batch / CameraTracker.TrackFrameBatch / Relocalize on the GPU: one live frame tracked against many
keyframes in lockstep must give, for every keyframe, bit for bit what dfk_se3_track gives for it alone on a fresh handle.
Inputs: the reference's 1047 -> 1052 tracking pair (tests/helpers.py) as a 3-level pyramid at 10/5/4 iterations."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import se3, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITERS = (10, 5, 4)
F = C.POINTER(C.c_float)
SENTINEL = np.float32(-7.25)  # what "left untouched" looks like


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def upload(torch, arr, extra_px=0):
    """host [H, W(, K)] -> device view whose rows are padded by extra_px pixels"""
    a = np.ascontiguousarray(arr, dtype=np.float32)
    h, w = a.shape[:2]
    k = a.shape[2] if a.ndim == 3 else 1
    row = (w + extra_px) * k
    buf = torch.zeros((h, row), dtype=torch.float32, device="cuda")
    buf[:, :w * k] = torch.from_numpy(a.reshape(h, w * k)).cuda()
    return buf[:, :w] if a.ndim == 2 else torch.as_strided(buf, (h, w, k), (row, k, 1))


class Problem:
    """one keyframe pyramid + the live frame + cameras + start pose, as DfkTrackLevel structs"""

    def __init__(self, torch, cams, p0, pd, p1, pg, pose, extra_px=0, iters=ITERS):
        self.cams, self.pose, self.iters = cams, np.asarray(pose, np.float32), tuple(iters)
        self.dev = [(upload(torch, p0[l], extra_px), upload(torch, pd[l], extra_px), upload(torch, p1[l], extra_px),
                     upload(torch, pg[l], extra_px)) for l in range(len(cams))]

    def levels(self, iters=None):
        from deepfactors_b200._lib import DfkTrackLevel
        from deepfactors_b200.aligners import _cam, _image
        iters = self.iters if iters is None else iters
        out = []
        for l, (i0, d0, i1, g1) in enumerate(self.dev):
            lv = DfkTrackLevel()
            lv.cam, lv.img0, lv.dpt0, lv.img1, lv.grad1 = _cam(self.cams[l]), _image(i0), _image(d0), _image(i1), _image(g1, 2)
            lv.iterations = int(iters[l])
            out.append(lv)
        return out


def handle():
    from deepfactors_b200.aligners import _Handle
    hd = _Handle()
    hd.use_torch_stream()
    return hd


def track_single(prob, hd=None, iters=None):
    """dfk_se3_track on a fresh handle (or `hd`): (pose, inlier fraction, error, last system)"""
    from deepfactors_b200._lib import DfkTrackLevel, check, lib
    hd = hd or handle()
    lv = prob.levels(iters)
    arr = (DfkTrackLevel * len(lv))(*lv)
    pose = prob.pose.copy()
    frac, err = np.full(1, SENTINEL), np.full(1, SENTINEL)
    sys_ = np.zeros(29, np.float32)
    check(hd.h, lib().dfk_se3_track(hd.h, pose.ctypes.data_as(F), arr, len(lv), frac.ctypes.data_as(F),
                                    err.ctypes.data_as(F), sys_.ctypes.data_as(F), None, 0))
    return pose, frac[0], err[0], sys_


def call_batch(hd, probs, iters=None):
    """dfk_se3_track_batch: (status, poses [N,7], fractions [N], errors [N], systems [N,29])"""
    from deepfactors_b200._lib import DfkTrackLevel, lib
    L = len(probs[0].cams)
    flat = [lv for p, it in zip(probs, iters or [None] * len(probs)) for lv in p.levels(it)]
    arr = (DfkTrackLevel * len(flat))(*flat)
    poses = np.ascontiguousarray(np.stack([p.pose for p in probs]), dtype=np.float32)
    n = len(probs)
    frac, err = np.full(n, SENTINEL), np.full(n, SENTINEL)
    sys_ = np.zeros((n, 29), np.float32)
    st = lib().dfk_se3_track_batch(hd.h, n, L, poses.ctypes.data_as(F), arr, frac.ctypes.data_as(F),
                                   err.ctypes.data_as(F), sys_.ctypes.data_as(F))
    return st, poses, frac, err, sys_


def track_batch(hd, probs, iters=None):
    from deepfactors_b200._lib import check
    st, *out = call_batch(hd, probs, iters)
    check(hd.h, st)
    return out


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_same(batch_out, n, single, what):
    poses, frac, err, sys_ = batch_out
    p, f, e, s = single
    assert np.array_equal(bits(poses[n]), bits(p)), f"{what}: pose {poses[n]} vs {p}"
    assert bits(frac[n]) == bits(f), f"{what}: inlier fraction {frac[n]} vs {f}"
    assert bits(err[n]) == bits(e), f"{what}: error {err[n]} vs {e}"
    assert np.array_equal(bits(sys_[n]), bits(s)), f"{what}: last system"


@pytest.fixture(scope="module")
def scene(torch_mod, oracle, golden):
    """the problems of the bitwise tests: start poses, pitched views, a decoy and a cropped (smaller) pair"""
    torch = torch_mod
    from helpers import tracking_pyramid
    cams, p0, p1, pd, pg = tracking_pyramid(golden, oracle, 3)
    mir0 = [np.ascontiguousarray(a[:, ::-1]) for a in p0]   # decoy: 1047 mirrored left-right, with its mirrored depth
    mird = [np.ascontiguousarray(a[:, ::-1]) for a in pd]
    # crop: level-0 window 256 x 192 at (32, 24), halved per level, principal point moved with it
    crop = lambda lst, l: np.ascontiguousarray(lst[l][(24 >> l):(24 >> l) + (192 >> l), (32 >> l):(32 >> l) + (256 >> l)])
    ccams = [synth.Camera(c.fx, c.fy, c.u0 - (32 >> l), c.v0 - (24 >> l), float(256 >> l), float(192 >> l))
             for l, c in enumerate(cams)]
    far = se3.make_pose([0, 0, 0], [0, 0, -100.0])  # every keyframe point lands behind the live camera
    ident = se3.identity()
    probs = {
        "identity": Problem(torch, cams, p0, pd, p1, pg, ident),
        "perturbed_a": Problem(torch, cams, p0, pd, p1, pg, se3.make_pose([0.01, -0.02, 0.005], [0.02, 0.01, -0.03])),
        "perturbed_b": Problem(torch, cams, p0, pd, p1, pg, se3.make_pose([-0.015, 0.01, 0.0], [-0.03, 0.02, 0.04])),
        "far": Problem(torch, cams, p0, pd, p1, pg, far),
        "pitched": Problem(torch, cams, p0, pd, p1, pg, ident, extra_px=5),
        "decoy": Problem(torch, cams, mir0, mird, p1, pg, ident),
        "cropped": Problem(torch, ccams, [crop(p0, l) for l in range(3)], [crop(pd, l) for l in range(3)],
                           [crop(p1, l) for l in range(3)], [crop(pg, l) for l in range(3)], ident),
    }
    singles = {k: track_single(p) for k, p in probs.items()}
    return dict(cams=cams, p0=p0, p1=p1, pd=pd, pg=pg, mir0=mir0, mird=mird, probs=probs, singles=singles)


def test_batch_equals_single_tracking_bit_for_bit(scene):
    probs, singles = scene["probs"], scene["singles"]
    names = list(probs)
    out = track_batch(handle(), [probs[k] for k in names])
    for n, k in enumerate(names):
        assert_same(out, n, singles[k], k)
    # the no-overlap problem comes back untouched with error = +inf
    far = names.index("far")
    assert np.array_equal(out[0][far], probs["far"].pose) and out[2][far] == np.inf and out[1][far] == 0.0
    # and the others did track
    assert out[2][names.index("identity")] < 1e-2


def test_batch_of_one_and_zero_level0_iterations(scene):
    probs = scene["probs"]
    out = track_batch(handle(), [probs["perturbed_a"]])
    assert_same(out, 0, scene["singles"]["perturbed_a"], "N = 1")
    # no level-0 iteration: inlier fraction and error stay untouched, pose and last system still match
    iters = (0, 5, 4)
    names = ["identity", "cropped", "far"]
    out = track_batch(handle(), [probs[k] for k in names], [iters] * len(names))
    for n, k in enumerate(names):
        single = track_single(probs[k], iters=iters)
        assert single[1] == SENTINEL and single[2] == SENTINEL
        assert_same(out, n, single, f"{k}, level 0 without iterations")


def test_permuting_problems_permutes_outputs(scene):
    probs = scene["probs"]
    names = list(probs)
    hd = handle()
    out = track_batch(hd, [probs[k] for k in names])
    perm = np.random.default_rng(3).permutation(len(names))
    outp = track_batch(hd, [probs[names[i]] for i in perm])
    for a, b in zip(out, outp):
        assert np.array_equal(bits(a[perm]), bits(b))


def test_handle_state_single_and_batched_calls_interleave(scene):
    from deepfactors_b200._lib import DFK_ERR_INVALID_ARG
    probs, singles = scene["probs"], scene["singles"]
    hd = handle()
    assert_same([x[None] for x in track_single(probs["perturbed_b"], hd)], 0, singles["perturbed_b"], "single first")
    names = ["decoy", "identity", "cropped"]
    out = track_batch(hd, [probs[k] for k in names])
    for n, k in enumerate(names):
        assert_same(out, n, singles[k], f"batched after single: {k}")
    assert_same([x[None] for x in track_single(probs["pitched"], hd)], 0, singles["pitched"], "single after batched")
    # a rejected call (one problem on another schedule) changes nothing for the next one
    st, *_ = call_batch(hd, [probs["identity"], probs["perturbed_a"]], [ITERS, (10, 5, 3)])
    assert st == DFK_ERR_INVALID_ARG
    names = ["perturbed_a", "far", "identity", "perturbed_b"]
    out = track_batch(hd, [probs[k] for k in names])
    for n, k in enumerate(names):
        assert_same(out, n, singles[k], f"after a rejected call: {k}")


def test_relocalize_picks_the_true_keyframe(torch_mod, scene, oracle):
    torch = torch_mod
    from deepfactors_b200.aligners import CameraTracker, TrackerConfig
    cams, p0, p1, pd, pg = (scene[k] for k in ("cams", "p0", "p1", "pd", "pg"))
    up = lambda lst: [upload(torch, a) for a in lst]
    trk = CameraTracker(cams, TrackerConfig(pyramid_levels=3, iterations_per_level=ITERS, huber_delta=0.1))
    decoy = (up(scene["mir0"]), up(scene["mird"]))
    true_kf = (up(p0), up(pd))
    live_img, live_grad = up(p1), up(pg)
    idx, pose_wc, errors = trk.Relocalize([decoy, true_kf, decoy], live_img, live_grad)
    # the standalone errors, keyframe by keyframe: the winner is their first argmin, and it is the true keyframe
    standalone = [scene["singles"]["decoy"][2], scene["singles"]["identity"][2], scene["singles"]["decoy"][2]]
    assert np.array_equal(bits(errors), bits(standalone))
    assert idx == int(np.argmin(standalone)) == 1
    assert trk.GetError() == errors[1]
    assert np.array_equal(pose_wc, trk.GetPoseEstimate())
    o_pose, _, _, _ = oracle.se3_track(se3.identity(np.float64), cams, p0, p1, pd, pg, ITERS, 0.1)
    assert np.abs(trk.pose_ck_ - o_pose).max() <= 2e-4
    # the next frame continues from the relocalised pose
    before = trk.GetError()
    trk.TrackFrame(live_img, live_grad)
    assert trk.GetError() <= before * 1.0001
    # nothing overlaps (no valid depth anywhere): the first keyframe, at its own pose
    void = [upload(torch, np.full_like(a, -1.0)) for a in pd]
    wk0, wk1 = se3.make_pose([0, 0.1, 0], [1, 2, 3]), se3.make_pose([0.1, 0, 0], [4, 5, 6])
    idx, pose_wc, errors = trk.Relocalize([(true_kf[0], void, wk0), (true_kf[0], void, wk1)], live_img, live_grad)
    assert idx == 0 and np.all(np.isinf(errors))
    assert np.allclose(pose_wc, wk0, atol=1e-7) and np.array_equal(trk.pose_ck_, se3.identity())


def test_facade_track_levels_batch_binary():
    subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "cpp"), "-f", "track_batch.mk"], check=True,
                   capture_output=True)
    exe = os.path.join(ROOT, "tests", "cpp", "track_batch_test")
    out = subprocess.run([exe], check=True, capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert "TRACK_BATCH_TEST_OK" in out.stdout
