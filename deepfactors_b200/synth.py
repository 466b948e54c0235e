"""Deterministic synthetic keyframe/frame data of the shapes the hot path consumes (numpy only).

Follows SURVEY.md section 8(d): SceneNet pinhole camera (tests/testing_utils.h:34-40), smooth
band-limited images, a proximity map giving 2-4.7 m depth at avg_dpt = 2, an iid N(0, 0.02^2)
code Jacobian, and the test poses of tests/ut_sfmaligner.cpp:254-264.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List

import numpy as np

from . import se3


@dataclass
class Camera:
    """df::PinholeCamera<float> (sources/common/algorithm/pinhole_camera.h:43)."""
    fx: float
    fy: float
    u0: float
    v0: float
    width: float
    height: float

    @staticmethod
    def scenenet(w: int, h: int) -> "Camera":
        # tests/testing_utils.h:34-40 (float arithmetic; w/2 and h/2 are integer divisions there)
        fx = np.float32(w // 2) / np.float32(0.5773502691896257)
        fy = np.float32(h // 2) / np.float32(0.41421356237309503)
        return Camera(float(fx), float(fy), float(w // 2), float(h // 2), float(w), float(h))

    def resized(self, new_w: int, new_h: int) -> "Camera":
        # PinholeCamera::ResizeViewport (pinhole_camera_impl.h:113-124), float arithmetic
        xr = np.float32(new_w) / np.float32(self.width)
        yr = np.float32(new_h) / np.float32(self.height)
        return Camera(float(np.float32(self.fx) * xr), float(np.float32(self.fy) * yr),
                      float(np.float32(self.u0) * xr), float(np.float32(self.v0) * yr), float(new_w), float(new_h))


def camera_pyramid(cam: Camera, levels: int) -> List[Camera]:
    """df::CameraPyramid (sources/common/algorithm/camera_pyramid.h:35-48): halve per level."""
    cams = [cam]
    for _ in range(1, levels):
        prev = cams[-1]
        cams.append(prev.resized(int(prev.width) // 2, int(prev.height) // 2))
    return cams


def sobel_np(img: np.ndarray) -> np.ndarray:
    """Sobel/8 with clamped border, (gx, gy) interleaved [H, W, 2] (cu_image_proc.cpp:57-92)."""
    p = np.pad(img.astype(np.float32), 1, mode="edge")
    H, W = img.shape

    def s(dy, dx):
        return p[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]

    gx = (-s(-1, -1) + s(-1, 1) - 2 * s(0, -1) + 2 * s(0, 1) - s(1, -1) + s(1, 1)) / np.float32(8)
    gy = (-s(-1, -1) - 2 * s(-1, 0) - s(-1, 1) + s(1, -1) + 2 * s(1, 0) + s(1, 1)) / np.float32(8)
    return np.stack([gx, gy], axis=-1).astype(np.float32)


def _field(w, h, scale, phase):
    """sum of three sinusoids (periods 7..25 px at scale 1), values in [0, 1]"""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    return _field_at(x * scale, y * scale, phase)


def _field_at(x, y, phase):
    """the field of _field at level-0 pixel coordinates (x, y) (any shape, not only the pixel grid)"""
    f = (np.sin(2 * np.pi * x / 25.0 + 0.3 + phase) * np.cos(2 * np.pi * y / 19.0 + 1.1 - 0.5 * phase)
         + 0.7 * np.sin(2 * np.pi * (x + 0.6 * y) / 13.0 + 2.0 + 0.7 * phase)
         + 0.5 * np.cos(2 * np.pi * (0.4 * x - y) / 7.0 + 0.5 + 1.3 * phase))
    return (0.5 + f / 4.4).astype(np.float32)


@dataclass
class PairLevel:
    """Inputs of one SfmAligner::RunStep at one pyramid level (host arrays)."""
    cam: Camera
    img0: np.ndarray      # [H, W]
    img1: np.ndarray      # [H, W]
    grad1: np.ndarray     # [H, W, 2]
    prx_orig: np.ndarray  # [H, W]
    prx_jac: np.ndarray   # [H, W, C]
    dpt0: np.ndarray      # [H, W] depth decoded from `code`
    std0: np.ndarray      # [H, W] (dead input)
    width: int = 0
    height: int = 0

    def __post_init__(self):
        self.height, self.width = self.img0.shape

    @property
    def algorithmic_bytes(self) -> int:
        """SURVEY 8(d): (24 + 4C) bytes per pixel"""
        c = self.prx_jac.shape[2]
        return self.width * self.height * (24 + 4 * c)


@dataclass
class Pair:
    pose0: np.ndarray
    pose1: np.ndarray
    code: np.ndarray
    levels: List[PairLevel] = field(default_factory=list)


def reference_test_poses(dtype=np.float32):
    """tests/ut_sfmaligner.cpp:254-264: pose0 = I, pose1 = SE3(exp(0.1,0.1,0), (-0.5,-0.5,0))^-1."""
    pose0 = se3.identity(dtype)
    pose = se3.make_pose([0.1, 0.1, 0.0], [-0.5, -0.5, 0.0], np.float64)
    return pose0, se3.inverse(pose, dtype)


def make_level(w: int, h: int, code_size: int, *, scale: float = 1.0, seed: int = 0, code=None, avg_dpt: float = 2.0,
               cam: Camera | None = None, phase: float = 0.0, jac_sigma: float = 0.02) -> PairLevel:
    cam = cam or Camera.scenenet(w, h)
    img0 = _field(w, h, scale, 0.0 + phase)
    img1 = _field(w, h, scale, 0.35 + phase)
    grad1 = sobel_np(img1)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    prx_orig = (0.4 + 0.1 * np.sin(x * scale / 20.0 + phase) * np.cos(y * scale / 25.0)).astype(np.float32)
    rng = np.random.default_rng(seed)
    prx_jac = (rng.standard_normal((h, w, code_size)) * jac_sigma).astype(np.float32)
    if code is None:
        code = np.zeros(code_size, dtype=np.float32)
    code = np.asarray(code, dtype=np.float32)
    prx = prx_orig + (prx_jac @ code).astype(np.float32)
    dpt0 = (np.float32(avg_dpt) / prx - np.float32(avg_dpt)).astype(np.float32)
    std0 = np.zeros((h, w), dtype=np.float32)
    return PairLevel(cam, img0, img1, grad1, prx_orig, prx_jac, dpt0, std0)


def rotated_view(level: PairLevel, scale: float, omega, phase: float = 0.0) -> np.ndarray:
    """img0 of a make_level level (pyramid scale `scale`, field phase `phase`) seen by a camera at the same centre
    rotated by R = exp(omega): the view of a frame whose pose relative to the keyframe's is (R, 0).  A pure rotation
    maps pixels by a homography whatever the depth, and img0 is an analytic field, so the view is exact (no resampling).
    The frame's pose is pose0 retracted by [0, 0, 0, omega] (se3.retract)."""
    cam = level.cam
    R = se3.quat_to_matrix(se3.so3_exp(omega))
    v, u = np.mgrid[0:level.height, 0:level.width].astype(np.float64)
    d = np.stack([(u - cam.u0) / cam.fx, (v - cam.v0) / cam.fy, np.ones_like(u)], axis=-1) @ R.T  # R d, row-wise
    x = cam.fx * d[..., 0] / d[..., 2] + cam.u0
    y = cam.fy * d[..., 1] / d[..., 2] + cam.v0
    return _field_at(x * scale, y * scale, phase)


def make_pair(w: int = 640, h: int = 480, code_size: int = 32, levels: int = 4, *, seed: int = 0,
              code_sigma: float = 0.0, identity_pose: bool = False, phase: float = 0.0) -> Pair:
    """One keyframe/frame pair with an `levels`-level pyramid (level 0 = w x h)."""
    if identity_pose:
        pose0, pose1 = se3.identity(), se3.identity()
    else:
        pose0, pose1 = reference_test_poses()
    rng = np.random.default_rng(seed + 1000003)
    code = (rng.standard_normal(code_size) * code_sigma).astype(np.float32)
    cams = camera_pyramid(Camera.scenenet(w, h), levels)
    out = Pair(pose0, pose1, code)
    for lvl, cam in enumerate(cams):
        out.levels.append(make_level(int(cam.width), int(cam.height), code_size, scale=float(2 ** lvl),
                                     seed=seed * 16 + lvl, code=code, cam=cam, phase=phase))
    return out
