"""Host-side SE(3) helpers in the Sophus conventions the reference uses.

A pose is a length-7 array in `Sophus::SE3f::data()` order: unit quaternion (x, y, z, w) then
translation (x, y, z).  The update model is the reference's (sources/core/gtsam/gtsam_traits.h:48-58,
tests/testing_utils.h:72-88, sources/common/algorithm/lucas_kanade_se3.h:84-95): translation
additive, rotation left-multiplied, `exp(w) * R`.
"""
from __future__ import annotations

import numpy as np


def identity(dtype=np.float32) -> np.ndarray:
    return np.array([0, 0, 0, 1, 0, 0, 0], dtype=dtype)


def quat_mul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([
        aw * bx + ax * bw + ay * bz - az * by,
        aw * by + ay * bw + az * bx - ax * bz,
        aw * bz + az * bw + ax * by - ay * bx,
        aw * bw - ax * bx - ay * by - az * bz,
    ])


def quat_rotate(q, v):
    qv = np.asarray(q[:3], dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    uv = 2.0 * np.cross(qv, v)
    return v + q[3] * uv + np.cross(qv, uv)


def quat_to_matrix(q):
    x, y, z, w = (float(c) for c in q)
    return np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
        [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
        [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)],
    ])


def so3_exp(omega) -> np.ndarray:
    """Sophus::SO3::exp -> quaternion (x, y, z, w)."""
    omega = np.asarray(omega, dtype=np.float64)
    theta_sq = float(omega @ omega)
    theta = np.sqrt(theta_sq)
    if theta < 1e-10:
        imag = 0.5 - theta_sq / 48.0 + theta_sq * theta_sq / 3840.0
        real = 1.0 - theta_sq / 8.0 + theta_sq * theta_sq / 384.0
    else:
        imag = np.sin(0.5 * theta) / theta
        real = np.cos(0.5 * theta)
    return np.array([imag * omega[0], imag * omega[1], imag * omega[2], real])


def make_pose(omega, trs, dtype=np.float32) -> np.ndarray:
    """Sophus::SE3(SO3::exp(omega), trs)."""
    return np.concatenate([so3_exp(omega), np.asarray(trs, dtype=np.float64)]).astype(dtype)


def inverse(pose, dtype=None) -> np.ndarray:
    p = np.asarray(pose, dtype=np.float64)
    qi = np.array([-p[0], -p[1], -p[2], p[3]])
    t = -quat_rotate(qi, p[4:7])
    return np.concatenate([qi, t]).astype(dtype or np.asarray(pose).dtype)


def compose(a, b, dtype=None) -> np.ndarray:
    a64 = np.asarray(a, dtype=np.float64)
    b64 = np.asarray(b, dtype=np.float64)
    q = quat_mul(a64[:4], b64[:4])
    q /= np.linalg.norm(q)
    t = a64[4:7] + quat_rotate(a64[:4], b64[4:7])
    return np.concatenate([q, t]).astype(dtype or np.asarray(a).dtype)


def retract(pose, delta, dtype=None) -> np.ndarray:
    """translation += delta[:3]; rotation = exp(delta[3:]) * rotation (gtsam_traits.h:48-58)."""
    p = np.asarray(pose, dtype=np.float64)
    d = np.asarray(delta, dtype=np.float64)
    q = quat_mul(so3_exp(d[3:6]), p[:4])
    q /= np.linalg.norm(q)
    return np.concatenate([q, p[4:7] + d[:3]]).astype(dtype or np.asarray(pose).dtype)


def so3_log(q) -> np.ndarray:
    """Sophus::SO3::log of a unit quaternion (x, y, z, w): the rotation vector omega with so3_exp(omega) = +-q."""
    q = np.asarray(q, dtype=np.float64)
    v, w = q[:3], float(q[3])
    n = float(np.linalg.norm(v))
    if n < 1e-10:
        scale = 2.0 / w - (2.0 / 3.0) * n * n / (w * w * w)
    else:
        # atan of the half angle kept in (-pi/2, pi/2]: the shortest rotation for q and -q alike
        scale = 2.0 * (np.arctan(n / w) if w != 0 else np.copysign(0.5 * np.pi, 1.0)) / n
    return scale * v


def local(pose0, pose, dtype=np.float64) -> np.ndarray:
    """The inverse of retract (gtsam_traits.h:66-72): delta = [t - t0 | log(R R0^T)], so retract(pose0, delta) = pose."""
    p0 = np.asarray(pose0, dtype=np.float64)
    p = np.asarray(pose, dtype=np.float64)
    q0i = np.array([-p0[0], -p0[1], -p0[2], p0[3]])
    return np.concatenate([p[4:7] - p0[4:7], so3_log(quat_mul(p[:4], q0i))]).astype(dtype)


def perturb(pose, idx: int, eps: float, dtype=None) -> np.ndarray:
    """tests/testing_utils.h:72-88 GetPerturbedPose."""
    d = np.zeros(6)
    d[idx] = eps
    return retract(pose, d, dtype)


def se3_solve_and_update(JtJ_dense, Jtr, pose) -> np.ndarray:
    """lucas_kanade_se3.h:84-95 SE3SolveAndUpdate: update = -JtJ.ldlt().solve(Jtr)."""
    H = np.asarray(JtJ_dense, dtype=np.float64)
    g = np.asarray(Jtr, dtype=np.float64)
    upd = -np.linalg.solve(H, g)
    return retract(pose, upd)
