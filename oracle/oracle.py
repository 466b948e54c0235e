"""ctypes front-end of the CPU oracle (oracle/libdfk_oracle.so).

TEST INFRASTRUCTURE ONLY -- see oracle/dfk_oracle.h.  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / `--impl reference` legs may import this module.  PARITY
UNPINNED: the reference cannot be built here (Eigen/Sophus/VisionCore absent) and ships no
golden vectors; see the header of dfk_oracle.h.

All arrays are numpy float32, C-contiguous rows; `pitch` is derived from strides and counted in
floats.  Images are [H, W]; grad1 is [H, W, 2]; prx_jac is [H, W, C].
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libdfk_oracle.so")


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (gcc, -O2 -ffp-contract=off)."""
    if force or not os.path.exists(_LIB_PATH) or any(
        os.path.getmtime(os.path.join(_HERE, f)) > os.path.getmtime(_LIB_PATH)
        for f in ("dfk_oracle.c", "dfk_oracle_impl.inc", "dfk_oracle.h", "Makefile")
    ):
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


class Camera(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("u0", C.c_float), ("v0", C.c_float),
                ("width", C.c_float), ("height", C.c_float)]


class SfmParams(C.Structure):
    _fields_ = [("huber_delta", C.c_float), ("ocl_th", C.c_float), ("avg_dpt", C.c_float),
                ("min_dpt", C.c_float), ("valid_border", C.c_int)]


def default_params(**kw) -> SfmParams:
    p = SfmParams(0.1, 1000.0, 2.0, 0.0, 2)  # dense_sfm.h:36-43
    for k, v in kw.items():
        setattr(p, k, v)
    return p


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.dfko_omp_max_threads.restype = C.c_int
        _lib.dfko_squared_error_f.restype = C.c_float
        _lib.dfko_squared_error_d.restype = C.c_double
    return _lib


def _f32(a):
    a = np.asarray(a)
    assert a.dtype == np.float32, a.dtype
    return a


def _ptr(a, ctype=C.c_float):
    return a.ctypes.data_as(C.POINTER(ctype))


def _pitch(a):
    """row pitch in floats of an [H, W(, K)] array whose rows are contiguous"""
    assert a.strides[-1] == a.itemsize
    if a.ndim == 3:
        assert a.strides[1] == a.itemsize * a.shape[2]
    assert a.strides[0] % a.itemsize == 0
    return C.c_size_t(a.strides[0] // a.itemsize)


def _cam(cam) -> Camera:
    if isinstance(cam, Camera):
        return cam
    return Camera(cam.fx, cam.fy, cam.u0, cam.v0, cam.width, cam.height)


@dataclass
class StepResult:
    JtJ: np.ndarray  # packed upper, NP(NP+1)/2
    Jtr: np.ndarray
    residual: float
    inliers: int

    @property
    def NP(self):
        return self.Jtr.shape[0]

    def dense(self) -> np.ndarray:
        n = self.NP
        H = np.zeros((n, n), dtype=self.JtJ.dtype)
        H[np.triu_indices(n)] = self.JtJ
        return H + np.triu(H, 1).T


def so3_exp(omega, dtype=np.float64):
    omega = np.ascontiguousarray(omega, dtype=dtype)
    q = np.zeros(4, dtype=dtype)
    fn = lib().dfko_so3_exp_d if dtype == np.float64 else lib().dfko_so3_exp_f
    ct = C.c_double if dtype == np.float64 else C.c_float
    fn(_ptr(omega, ct), _ptr(q, ct))
    return q


def pose_perturb(pose, idx, eps, dtype=np.float64):
    pose = np.ascontiguousarray(pose, dtype=dtype)
    out = np.zeros(7, dtype=dtype)
    if dtype == np.float64:
        lib().dfko_pose_perturb_d(_ptr(pose, C.c_double), C.c_int(idx), C.c_double(eps), _ptr(out, C.c_double))
    else:
        lib().dfko_pose_perturb_f(_ptr(pose, C.c_float), C.c_int(idx), C.c_float(eps), _ptr(out, C.c_float))
    return out


def relative_pose(a, b, dtype=np.float64, jacobians=True):
    a = np.ascontiguousarray(a, dtype=dtype)
    b = np.ascontiguousarray(b, dtype=dtype)
    ab = np.zeros(7, dtype=dtype)
    ja = np.zeros(36, dtype=dtype)
    jb = np.zeros(36, dtype=dtype)
    ct = C.c_double if dtype == np.float64 else C.c_float
    fn = lib().dfko_relative_pose_d if dtype == np.float64 else lib().dfko_relative_pose_f
    fn(_ptr(a, ct), _ptr(b, ct), _ptr(ab, ct), _ptr(ja, ct) if jacobians else None, _ptr(jb, ct) if jacobians else None)
    return ab, ja.reshape(6, 6), jb.reshape(6, 6)


def probe_pixel(x, y, dpt, cam, pose, border=1, min_dpt=0.0, avg_dpt=2.0):
    pose = np.ascontiguousarray(pose, dtype=np.float64)
    out = np.zeros(17, dtype=np.float64)
    c = _cam(cam)
    lib().dfko_probe_pixel_d(C.c_double(x), C.c_double(y), C.c_double(dpt), C.byref(c), _ptr(pose, C.c_double),
                             C.c_int(border), C.c_double(min_dpt), C.c_double(avg_dpt), _ptr(out, C.c_double))
    return dict(valid=bool(out[0]), pix1=out[1:3].copy(), J_pose=out[3:15].reshape(2, 6).copy(),
                J_prx=out[15:17].copy())


def sfm_run_step(pose0, pose1, cam, img0, img1, dpt0, valid0, prx0_jac, grad1, params=None, *,
                 precision="f32", loop_order=0, omp_threads=None) -> StepResult:
    """SfmAligner::RunStep on the CPU.  precision: "f32" (reference-like) or "f64" (truth).
    omp_threads: if not None, use the OpenMP row-major float variant (CPU baseline)."""
    params = params or default_params()
    img0, img1, dpt0, prx0_jac, grad1 = map(_f32, (img0, img1, dpt0, prx0_jac, grad1))
    H, W = img0.shape
    Cs = prx0_jac.shape[2]
    assert prx0_jac.shape[:2] == (H, W) and grad1.shape == (H, W, 2)
    NP = 12 + Cs
    pose0 = np.ascontiguousarray(pose0, dtype=np.float32)
    pose1 = np.ascontiguousarray(pose1, dtype=np.float32)
    c = _cam(cam)
    inl = C.c_uint64(0)
    vptr, vpitch = (None, C.c_size_t(0)) if valid0 is None else (_ptr(_f32(valid0)), _pitch(valid0))
    common = (_ptr(pose0), _ptr(pose1), C.c_int(Cs), C.byref(c), C.c_int(W), C.c_int(H),
              _ptr(img0), _pitch(img0), _ptr(img1), _pitch(img1), _ptr(dpt0), _pitch(dpt0), vptr, vpitch,
              _ptr(prx0_jac), _pitch(prx0_jac), _ptr(grad1), _pitch(grad1), C.byref(params))
    if precision == "f64":
        JtJ = np.zeros(NP * (NP + 1) // 2, dtype=np.float64)
        Jtr = np.zeros(NP, dtype=np.float64)
        res = C.c_double(0)
        lib().dfko_sfm_run_step_d(*common, C.c_int(loop_order), _ptr(JtJ, C.c_double), _ptr(Jtr, C.c_double),
                                  C.byref(res), C.byref(inl))
    else:
        JtJ = np.zeros(NP * (NP + 1) // 2, dtype=np.float32)
        Jtr = np.zeros(NP, dtype=np.float32)
        res = C.c_float(0)
        if omp_threads is not None:
            lib().dfko_sfm_run_step_f_omp(*common, C.c_int(omp_threads), _ptr(JtJ), _ptr(Jtr), C.byref(res),
                                          C.byref(inl))
        else:
            lib().dfko_sfm_run_step_f(*common, C.c_int(loop_order), _ptr(JtJ), _ptr(Jtr), C.byref(res), C.byref(inl))
    return StepResult(JtJ, Jtr, float(res.value), int(inl.value))


def sfm_pixel_rows(pose0, pose1, cam, img0, img1, dpt0, valid0, prx0_jac, grad1, params=None, *, y_begin=0,
                   y_end=None):
    """The fp64 per-pixel rows that sfm_run_step(..., precision="f64") sums, for image rows y_begin .. y_end-1.
    Returns (rows [(y_end - y_begin) * W, NP + 1] float64, row-major over the pixels: [J (NP) | w*diff], zero for an
    invalid pixel; residual of the range; inliers of the range).  valid0: None or the full [H, W] mask (in/out)."""
    params = params or default_params()
    img0, img1, dpt0, prx0_jac, grad1 = map(_f32, (img0, img1, dpt0, prx0_jac, grad1))
    H, W = img0.shape
    Cs = prx0_jac.shape[2]
    assert prx0_jac.shape[:2] == (H, W) and grad1.shape == (H, W, 2)
    y_end = H if y_end is None else min(int(y_end), H)
    y_begin = max(0, min(int(y_begin), y_end))
    NP = 12 + Cs
    pose0 = np.ascontiguousarray(pose0, dtype=np.float32)
    pose1 = np.ascontiguousarray(pose1, dtype=np.float32)
    c = _cam(cam)
    inl = C.c_uint64(0)
    res = C.c_double(0)
    rows = np.empty(((y_end - y_begin) * W, NP + 1), dtype=np.float64)
    vptr, vpitch = (None, C.c_size_t(0)) if valid0 is None else (_ptr(_f32(valid0)), _pitch(valid0))
    lib().dfko_sfm_pixel_rows_d(_ptr(pose0), _ptr(pose1), C.c_int(Cs), C.byref(c), C.c_int(W), C.c_int(H),
                                _ptr(img0), _pitch(img0), _ptr(img1), _pitch(img1), _ptr(dpt0), _pitch(dpt0), vptr,
                                vpitch, _ptr(prx0_jac), _pitch(prx0_jac), _ptr(grad1), _pitch(grad1), C.byref(params),
                                C.c_int(y_begin), C.c_int(y_end), _ptr(rows, C.c_double), C.byref(res), C.byref(inl))
    return rows, float(res.value), int(inl.value)


def sfm_evaluate_error(pose0, pose1, cam, img0, img1, dpt0, params=None, *, precision="f32"):
    params = params or default_params()
    img0, img1, dpt0 = map(_f32, (img0, img1, dpt0))
    H, W = img0.shape
    pose0 = np.ascontiguousarray(pose0, dtype=np.float32)
    pose1 = np.ascontiguousarray(pose1, dtype=np.float32)
    c = _cam(cam)
    inl = C.c_uint64(0)
    args = (_ptr(pose0), _ptr(pose1), C.byref(c), C.c_int(W), C.c_int(H), _ptr(img0), _pitch(img0), _ptr(img1),
            _pitch(img1), _ptr(dpt0), _pitch(dpt0), C.byref(params))
    if precision == "f64":
        res = C.c_double(0)
        lib().dfko_sfm_evaluate_error_d(*args, C.byref(res), C.byref(inl))
    else:
        res = C.c_float(0)
        lib().dfko_sfm_evaluate_error_f(*args, C.byref(res), C.byref(inl))
    return float(res.value), int(inl.value)


def se3_run_step(se3, cam, img0, img1, dpt0, grad1, huber_delta=0.1, *, precision="f32") -> StepResult:
    img0, img1, dpt0, grad1 = map(_f32, (img0, img1, dpt0, grad1))
    H, W = img0.shape
    se3 = np.ascontiguousarray(se3, dtype=np.float32)
    c = _cam(cam)
    inl = C.c_uint64(0)
    args = (_ptr(se3), C.byref(c), C.c_int(W), C.c_int(H), _ptr(img0), _pitch(img0), _ptr(img1), _pitch(img1),
            _ptr(dpt0), _pitch(dpt0), _ptr(grad1), _pitch(grad1), C.c_float(huber_delta))
    if precision == "f64":
        JtJ = np.zeros(21, dtype=np.float64)
        Jtr = np.zeros(6, dtype=np.float64)
        res = C.c_double(0)
        lib().dfko_se3_run_step_d(*args, _ptr(JtJ, C.c_double), _ptr(Jtr, C.c_double), C.byref(res), C.byref(inl))
    else:
        JtJ = np.zeros(21, dtype=np.float32)
        Jtr = np.zeros(6, dtype=np.float32)
        res = C.c_float(0)
        lib().dfko_se3_run_step_f(*args, _ptr(JtJ), _ptr(Jtr), C.byref(res), C.byref(inl))
    return StepResult(JtJ, Jtr, float(res.value), int(inl.value))


def se3_warp(se3, cam, img0, img1, dpt0, *, precision="f32"):
    img0, img1, dpt0 = map(_f32, (img0, img1, dpt0))
    H, W = img0.shape
    se3 = np.ascontiguousarray(se3, dtype=np.float32)
    img2 = np.zeros((H, W), dtype=np.float32)
    c = _cam(cam)
    inl = C.c_uint64(0)
    args = (_ptr(se3), C.byref(c), C.c_int(W), C.c_int(H), _ptr(img0), _pitch(img0), _ptr(img1), _pitch(img1),
            _ptr(dpt0), _pitch(dpt0), _ptr(img2), _pitch(img2))
    if precision == "f64":
        res = C.c_double(0)
        lib().dfko_se3_warp_d(*args, C.byref(res), C.byref(inl))
    else:
        res = C.c_float(0)
        lib().dfko_se3_warp_f(*args, C.byref(res), C.byref(inl))
    return img2, float(res.value), int(inl.value)


def se3_track(pose_ck, cams, pyr_img0, pyr_img1, pyr_dpt0, pyr_grad1, iterations_per_level, huber_delta=0.1, *,
              precision="f64"):
    """CameraTracker::TrackFrame (core/system/camera_tracker.cpp:42-69): levels coarse -> fine, per iteration
    SE3Aligner::RunStep, update = -JtJ.ldlt().solve(Jtr), t += update[:3], so3 = exp(update[3:]) * so3.
    Returns (pose, inlier_fraction, error, history) with history[i] = (StepResult, pose it was evaluated at)."""
    pose = np.asarray(pose_ck, dtype=np.float64).copy()
    hist = []
    frac, err = 0.0, float("inf")
    for level in range(len(cams) - 1, -1, -1):
        for _ in range(int(iterations_per_level[level])):
            r = se3_run_step(pose.astype(np.float32), cams[level], pyr_img0[level], pyr_img1[level], pyr_dpt0[level],
                             pyr_grad1[level], huber_delta, precision=precision)
            hist.append((r, pose.copy()))
            frac = r.inliers / float(pyr_img1[level].shape[0] * pyr_img1[level].shape[1])
            err = r.residual / r.inliers if r.inliers else float("inf")
            if r.inliers == 0:
                continue
            Hd = np.zeros((6, 6))
            Hd[np.triu_indices(6)] = np.asarray(r.JtJ, dtype=np.float64)
            Hd = Hd + np.triu(Hd, 1).T
            upd = -np.linalg.solve(Hd, np.asarray(r.Jtr, dtype=np.float64))
            dq = so3_exp(upd[3:6])
            x1, y1, z1, w1 = dq
            x2, y2, z2, w2 = pose[:4]
            q = np.array([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                          w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2])
            pose = np.concatenate([q / np.linalg.norm(q), pose[4:7] + upd[:3]])
    return pose, frac, err, hist


def update_depth(code, prx_orig, prx_jac, avg_dpt=2.0):
    code = np.ascontiguousarray(code, dtype=np.float32)
    prx_orig, prx_jac = _f32(prx_orig), _f32(prx_jac)
    H, W = prx_orig.shape
    out = np.zeros((H, W), dtype=np.float32)
    lib().dfko_update_depth_f(_ptr(code), C.c_int(code.shape[0]), C.c_int(W), C.c_int(H), _ptr(prx_orig),
                              _pitch(prx_orig), _ptr(prx_jac), _pitch(prx_jac), C.c_float(avg_dpt), _ptr(out),
                              _pitch(out))
    return out


def depth_run_step(code, target_dpt, prx_orig, prx_jac, avg_dpt=2.0, *, precision="f32") -> StepResult:
    """DepthAligner::RunStep on the CPU (cu_depthaligner.cpp:32-113)."""
    code = np.ascontiguousarray(code, dtype=np.float32)
    tgt, prx_orig, prx_jac = _f32(target_dpt), _f32(prx_orig), _f32(prx_jac)
    H, W = tgt.shape
    Cs = code.shape[0]
    inl = C.c_uint64(0)
    args = (_ptr(code), C.c_int(Cs), C.c_int(W), C.c_int(H), _ptr(tgt), _pitch(tgt), _ptr(prx_orig), _pitch(prx_orig),
            _ptr(prx_jac), _pitch(prx_jac), C.c_float(avg_dpt))
    if precision == "f64":
        JtJ, Jtr, res = np.zeros(Cs * (Cs + 1) // 2), np.zeros(Cs), C.c_double(0)
        lib().dfko_depth_run_step_d(*args, _ptr(JtJ, C.c_double), _ptr(Jtr, C.c_double), C.byref(res), C.byref(inl))
    else:
        JtJ, Jtr, res = np.zeros(Cs * (Cs + 1) // 2, dtype=np.float32), np.zeros(Cs, dtype=np.float32), C.c_float(0)
        lib().dfko_depth_run_step_f(*args, _ptr(JtJ), _ptr(Jtr), C.byref(res), C.byref(inl))
    return StepResult(JtJ, Jtr, float(res.value), int(inl.value))


def reprojection_rows(pose0, pose1, code, cam, prx_orig, prx_jac, query_xy, train_xy, cauchy_delta, sigma, avg_dpt=2.0, *,
                      precision="f32"):
    """ReprojectionFactor::linearize rows on the CPU (reprojection_factor.cpp:157-269).  Returns (rows [2M, 13+C], total_err)."""
    code = np.ascontiguousarray(code, dtype=np.float32)
    prx_orig, prx_jac = _f32(prx_orig), _f32(prx_jac)
    H, W = prx_orig.shape
    Cs = code.shape[0]
    q = np.ascontiguousarray(query_xy, dtype=np.float32).reshape(-1, 2)
    t = np.ascontiguousarray(train_xy, dtype=np.float32).reshape(-1, 2)
    M = q.shape[0]
    pose0 = np.ascontiguousarray(pose0, dtype=np.float32)
    pose1 = np.ascontiguousarray(pose1, dtype=np.float32)
    c = _cam(cam)
    dt, ct = (np.float64, C.c_double) if precision == "f64" else (np.float32, C.c_float)
    rows = np.zeros((2 * M, 13 + Cs), dtype=dt)
    fn = lib().dfko_reprojection_rows_d if precision == "f64" else lib().dfko_reprojection_rows_f
    fn.restype = ct
    tot = fn(_ptr(pose0), _ptr(pose1), _ptr(code), C.c_int(Cs), C.byref(c), C.c_int(W), C.c_int(H), _ptr(prx_orig),
             _pitch(prx_orig), _ptr(prx_jac), _pitch(prx_jac), C.c_int(M), _ptr(q), _ptr(t), C.c_float(cauchy_delta),
             C.c_float(sigma), C.c_float(avg_dpt), _ptr(rows, ct))
    return rows, float(tot)


def sparse_geometric_rows(pose0, pose1, code0, code1, cam, prx0_orig, prx0_jac, prx1_orig, prx1_jac, dpt_grad1, points_xy,
                          huber_delta, avg_dpt=2.0, *, precision="f32"):
    """SparseGeometricFactor::linearize rows on the CPU (sparse_geometric_factor.cpp:157-271).
    Returns (rows [M, 13 + 2C], number of valid rows)."""
    code0 = np.ascontiguousarray(code0, dtype=np.float32)
    code1 = np.ascontiguousarray(code1, dtype=np.float32)
    prx0_orig, prx0_jac, prx1_orig, prx1_jac, dpt_grad1 = map(_f32, (prx0_orig, prx0_jac, prx1_orig, prx1_jac, dpt_grad1))
    H, W = prx0_orig.shape
    Cs = code0.shape[0]
    pts = np.ascontiguousarray(points_xy, dtype=np.int32).reshape(-1, 2)
    M = pts.shape[0]
    pose0 = np.ascontiguousarray(pose0, dtype=np.float32)
    pose1 = np.ascontiguousarray(pose1, dtype=np.float32)
    c = _cam(cam)
    dt, ct = (np.float64, C.c_double) if precision == "f64" else (np.float32, C.c_float)
    rows = np.zeros((M, 13 + 2 * Cs), dtype=dt)
    fn = lib().dfko_sparse_geometric_rows_d if precision == "f64" else lib().dfko_sparse_geometric_rows_f
    fn.restype = C.c_int
    n = fn(_ptr(pose0), _ptr(pose1), _ptr(code0), _ptr(code1), C.c_int(Cs), C.byref(c), C.c_int(W), C.c_int(H),
           _ptr(prx0_orig), _pitch(prx0_orig), _ptr(prx0_jac), _pitch(prx0_jac), _ptr(prx1_orig), _pitch(prx1_orig),
           _ptr(prx1_jac), _pitch(prx1_jac), _ptr(dpt_grad1), _pitch(dpt_grad1), C.c_int(M),
           pts.ctypes.data_as(C.POINTER(C.c_int)), C.c_float(huber_delta), C.c_float(avg_dpt), _ptr(rows, ct))
    return rows, int(n)


def sobel_gradients(img):
    img = _f32(img)
    H, W = img.shape
    grad = np.zeros((H, W, 2), dtype=np.float32)
    lib().dfko_sobel_gradients_f(C.c_int(W), C.c_int(H), _ptr(img), _pitch(img), _ptr(grad), _pitch(grad))
    return grad


def gaussian_blur_down(img):
    img = _f32(img)
    H, W = img.shape
    out = np.zeros((H // 2, W // 2), dtype=np.float32)  # camera_pyramid.h:43-44 integer halving
    lib().dfko_gaussian_blur_down_f(C.c_int(W), C.c_int(H), _ptr(img), _pitch(img), C.c_int(W // 2), C.c_int(H // 2),
                                    _ptr(out), _pitch(out))
    return out


def squared_error(a, b, precision="f32"):
    a, b = _f32(a), _f32(b)
    H, W = a.shape
    fn = lib().dfko_squared_error_d if precision == "f64" else lib().dfko_squared_error_f
    return float(fn(C.c_int(W), C.c_int(H), _ptr(a), _pitch(a), _ptr(b), _pitch(b)))


class Level(C.Structure):
    """DfkoLevel / RefLevel: one pyramid level of a pair for the throughput-mode CPU baselines"""
    _fields_ = [("cam", Camera), ("width", C.c_int), ("height", C.c_int),
                ("img0", C.POINTER(C.c_float)), ("img0_pitch", C.c_size_t),
                ("img1", C.POINTER(C.c_float)), ("img1_pitch", C.c_size_t),
                ("dpt0", C.POINTER(C.c_float)), ("dpt0_pitch", C.c_size_t),
                ("prx0_jac", C.POINTER(C.c_float)), ("jac_pitch", C.c_size_t),
                ("grad1", C.POINTER(C.c_float)), ("grad1_pitch", C.c_size_t)]


def make_levels(levels):
    """levels: objects with cam, img0, img1, dpt0, prx_jac, grad1 (deepfactors_b200.synth.PairLevel).  Returns the
    ctypes array and the list of arrays it points into (keep both alive)."""
    arr = (Level * len(levels))()
    keep = []
    for i, L in enumerate(levels):
        a = [np.ascontiguousarray(_f32(x)) for x in (L.img0, L.img1, L.dpt0, L.prx_jac, L.grad1)]
        keep.append(a)
        H, W = a[0].shape
        arr[i] = Level(_cam(L.cam), W, H, _ptr(a[0]), _pitch(a[0]), _ptr(a[1]), _pitch(a[1]), _ptr(a[2]), _pitch(a[2]),
                       _ptr(a[3]), _pitch(a[3]), _ptr(a[4]), _pitch(a[4]))
    return arr, keep


def sfm_throughput(pose0, pose1, levels, nthreads, evals_per_thread, params=None, loop_order=1):
    """`nthreads` POSIX threads x `evals_per_thread` whole-pyramid evaluations (single-threaded dfko_sfm_run_step_f
    each).  Returns (wall seconds, StepResult of level 0 from thread 0)."""
    params = params or default_params()
    arr, keep = make_levels(levels)
    Cs = keep[0][3].shape[2]
    NP = 12 + Cs
    NH = NP * (NP + 1) // 2
    rec = np.zeros(NH + NP + 2, dtype=np.float32)
    pose0 = np.ascontiguousarray(pose0, dtype=np.float32)
    pose1 = np.ascontiguousarray(pose1, dtype=np.float32)
    fn = lib().dfko_sfm_throughput_f
    fn.restype = C.c_double
    dt = fn(C.c_int(nthreads), C.c_int(evals_per_thread), C.c_int(loop_order), _ptr(pose0), _ptr(pose1), C.c_int(Cs),
            C.c_int(len(levels)), arr, C.byref(params), _ptr(rec))
    return float(dt), StepResult(rec[:NH].copy(), rec[NH:NH + NP].copy(), float(rec[NH + NP]), int(rec[NH + NP + 1]))


def omp_max_threads() -> int:
    return int(lib().dfko_omp_max_threads())
