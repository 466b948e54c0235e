"""CPU tests of CameraTracker.Relocalize's host side: the selection rule of DeepFactors::Relocalize
(core/deepfactors.cpp:717-733) and the argument checks of TrackFrameBatch.  No GPU needed."""
import numpy as np
import pytest

from deepfactors_b200 import se3
from deepfactors_b200.aligners import CameraTracker, batch_start_poses, relocalize_select

INF = float("inf")


def poses(n, seed=0):
    rng = np.random.default_rng(seed)
    return np.stack([se3.make_pose(rng.normal(0, 0.1, 3), rng.normal(0, 0.5, 3)) for _ in range(n)])


def estimate(pose_wk, pose_ck):
    """CameraTracker.GetPoseEstimate of a tracker whose keyframe pose is pose_wk and pose_ck_ = pose_ck"""
    trk = CameraTracker.__new__(CameraTracker)  # the pose algebra only, no device handle
    trk.kf_ = (None, None, None if pose_wk is None else np.asarray(pose_wk, np.float32))
    trk.pose_ck_ = np.asarray(pose_ck, np.float32)
    return trk.GetPoseEstimate()


@pytest.mark.parametrize("errors, want", [
    ([0.5, 0.2, 0.3], 1),
    ([0.2, 0.2, 0.1, 0.1], 2),          # ties: the first of the smallest (strict <)
    ([0.3, 0.3, 0.3], 0),
    ([INF, 0.4, INF], 1),
    ([float("nan"), 0.4, 0.4], 1),      # NaN never compares smaller
    ([0.1], 0),
])
def test_first_strict_minimum(errors, want):
    pck, pwk = poses(len(errors)), poses(len(errors), seed=1)
    idx, pose_ck, pose_wc = relocalize_select(np.asarray(errors, np.float32), pck, list(pwk))
    assert idx == want
    assert np.array_equal(pose_ck, pck[want])
    assert np.array_equal(pose_wc, estimate(pwk[want], pck[want]))


def test_all_infinite_falls_back_to_the_first_keyframe_at_its_own_pose():
    pck, pwk = poses(3), poses(3, seed=1)
    idx, pose_ck, pose_wc = relocalize_select(np.full(3, np.inf, np.float32), pck, list(pwk))
    assert idx == 0
    assert np.array_equal(pose_ck, se3.identity())
    assert np.allclose(pose_wc, pwk[0], atol=1e-7)
    assert np.array_equal(pose_wc, estimate(pwk[0], se3.identity()))


def test_keyframes_without_a_world_pose_count_as_identity():
    pck = poses(2)
    idx, pose_ck, pose_wc = relocalize_select([0.3, 0.1], pck, [None, None])
    assert idx == 1 and np.array_equal(pose_wc, estimate(None, pck[1]))
    assert np.allclose(se3.compose(pose_wc, pose_ck), se3.identity(), atol=1e-6)


def test_batch_arguments_are_checked_before_any_device_work():
    lv = [object()] * 3
    assert batch_start_poses([(lv, lv)], 3).tolist() == [[0, 0, 0, 1, 0, 0, 0]]
    p = batch_start_poses([(lv, lv), (lv, lv, None)], 3, poses(2))
    assert p.shape == (2, 7) and p.dtype == np.float32 and p.flags.c_contiguous
    with pytest.raises(ValueError, match="1 to 65535"):
        batch_start_poses([], 3)
    with pytest.raises(ValueError, match="1 to 65535"):
        batch_start_poses([(lv, lv)] * 65536, 3)
    with pytest.raises(ValueError, match="keyframe 1 must be"):
        batch_start_poses([(lv, lv), (lv,)], 3)
    with pytest.raises(ValueError, match="keyframe 0 needs 3 pyramid levels"):
        batch_start_poses([(lv[:2], lv)], 3)
    with pytest.raises(ValueError, match="2 x 7"):
        batch_start_poses([(lv, lv), (lv, lv)], 3, poses(3))
    # the caller's start poses are copied, not updated in place
    start = poses(1)
    out = batch_start_poses([(lv, lv)], 3, start)
    out[0, 4] += 1.0
    assert not np.array_equal(out, start)
