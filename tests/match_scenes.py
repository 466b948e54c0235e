"""Synthetic two-view scenes for the keypoint matching tests: keypoints of known (R, t), pixel noise, injected outliers,
and binary descriptors whose Hamming matching pairs query q with train q."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class Cam:
    fx: float = 500.0
    fy: float = 500.0
    u0: float = 320.0
    v0: float = 240.0
    width: float = 640.0
    height: float = 480.0


def rodrigues(w) -> np.ndarray:
    w = np.asarray(w, np.float64)
    th = np.linalg.norm(w)
    if th == 0:
        return np.eye(3)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def rotation_angle(Ra, Rb) -> float:
    M = Ra.T @ Rb  # atan2 of the axis length and the cosine: accurate near 0, unlike arccos
    s = 0.5 * np.linalg.norm([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    return float(np.arctan2(s, (np.trace(M) - 1) / 2))


def bearing(xy, cam):
    x = (np.asarray(xy, np.float64)[:, 0] - cam.u0) / cam.fx
    y = (np.asarray(xy, np.float64)[:, 1] - cam.v0) / cam.fy
    f = np.stack([x, y, np.ones_like(x)], 1)
    return f / np.linalg.norm(f, axis=1, keepdims=True)


@dataclass
class Scene:
    cam: Cam
    R: np.ndarray
    t: np.ndarray
    kp0: np.ndarray        # [N, 2] float32
    kp1: np.ndarray        # [N, 2] float32: match q is (kp0[q], kp1[q])
    inlier: np.ndarray     # [N] bool: not an injected outlier
    desc0: np.ndarray      # [N, D] uint8
    desc1: np.ndarray      # [N, D] uint8, desc1[q] = desc0[q] with `flips[q]` bits flipped
    flips: np.ndarray      # [N] int: the Hamming distance of match q


def project(X, cam):
    return np.stack([cam.fx * X[:, 0] / X[:, 2] + cam.u0, cam.fy * X[:, 1] / X[:, 2] + cam.v0], 1)


def make_scene(n, outlier_frac, noise_px, seed, desc_bytes=32, cam=None, max_flips=24, outlier_margin=None) -> Scene:
    """n correspondences of points at depth 2-6 seen from two views (X1 = R X0 + t, rotation ~0.1 rad, baseline 0.3).
    outlier_frac of the matches get a random second keypoint; with outlier_margin, an outlier is redrawn until its
    score under the true (R, t) (the oracle's measure) is at least outlier_margin, so that it lies off its epipolar
    line: an outlier on the line cannot be told from an inlier by two-view geometry."""
    cam = cam or Cam()
    rng = np.random.default_rng(seed)
    R = rodrigues(rng.normal(size=3) * 0.06)
    t = rng.normal(size=3)
    t = 0.3 * t / np.linalg.norm(t)
    kp0, kp1 = [], []
    while len(kp0) < n:
        px = rng.uniform([0, 0], [cam.width, cam.height], (4 * n, 2))
        z = rng.uniform(2, 6, 4 * n)
        X0 = np.stack([(px[:, 0] - cam.u0) / cam.fx * z, (px[:, 1] - cam.v0) / cam.fy * z, z], 1)
        X1 = X0 @ R.T + t
        p1 = project(X1, cam)
        ok = (X1[:, 2] > 0.1) & (p1[:, 0] >= 0) & (p1[:, 0] < cam.width) & (p1[:, 1] >= 0) & (p1[:, 1] < cam.height)
        kp0 += list(px[ok])
        kp1 += list(p1[ok])
    kp0 = np.array(kp0[:n]) + rng.normal(scale=noise_px, size=(n, 2))
    kp1 = np.array(kp1[:n]) + rng.normal(scale=noise_px, size=(n, 2))
    inlier = np.ones(n, bool)
    out = rng.choice(n, int(round(outlier_frac * n)), replace=False)
    inlier[out] = False
    for q in out:
        while True:
            kp1[q] = rng.uniform([0, 0], [cam.width, cam.height])
            if outlier_margin is None:
                break
            from match_oracle import match_oracle as mo
            f0 = bearing(kp0[q:q + 1].astype(np.float32), cam)[0]
            f1 = bearing(kp1[q:q + 1].astype(np.float32), cam)[0]
            if mo.score(R, t, f0, f1) >= outlier_margin:
                break
    desc0 = rng.integers(0, 256, (n, desc_bytes), dtype=np.uint8)
    flips = rng.integers(0, max_flips + 1, n)
    bits = np.unpackbits(desc0, axis=1)
    for q in range(n):
        pos = rng.choice(bits.shape[1], flips[q], replace=False)
        bits[q, pos] ^= 1
    desc1 = np.packbits(bits, axis=1)
    return Scene(cam, R, t, kp0.astype(np.float32), kp1.astype(np.float32), inlier, desc0, desc1, flips)
