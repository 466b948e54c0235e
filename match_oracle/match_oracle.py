"""ctypes front-end of the keypoint-matching oracle (match_oracle/libdfk_match_oracle.so).

TEST INFRASTRUCTURE ONLY: tests/ and tools/bench_secondary.py use it as the checker of dfk_hamming_match_batch and
dfk_reprojection_match_batch.  Keypoints are float32 [N, 2], descriptors uint8 [N, D] (D = 32 or 64).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libdfk_match_oracle.so")
_MODEL = os.path.join(_HERE, "..", "deepfactors_b200", "csrc", "dfk_match_model.h")


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (gcc, -O2 -ffp-contract=off)."""
    srcs = [os.path.join(_HERE, f) for f in ("dfk_match_oracle.c", "Makefile")] + [_MODEL]
    if force or not os.path.exists(_LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(_LIB_PATH) for f in srcs):
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


class Params(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("u0", C.c_double), ("v0", C.c_double),
                ("threshold", C.c_double), ("probability", C.c_double), ("max_dist", C.c_float),
                ("max_iterations", C.c_int32), ("seed", C.c_uint64)]


_lib = None
_D = C.POINTER(C.c_double)
_I = C.POINTER(C.c_int32)


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.dfkm_hamming.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, _I]
        L.dfkm_sample.argtypes = [C.c_uint64, C.c_int, C.c_int, _I]
        L.dfkm_sample.restype = C.c_int
        L.dfkm_bearing.argtypes = [C.c_float, C.c_float, C.c_double, C.c_double, C.c_double, C.c_double, _D]
        L.dfkm_eightpt.argtypes = [_D, _D, _D]
        L.dfkm_eightpt.restype = C.c_int
        L.dfkm_model.argtypes = [_D, _D, _D, _D]
        L.dfkm_model.restype = C.c_int
        L.dfkm_score.argtypes = [_D, _D, _D, _D]
        L.dfkm_score.restype = C.c_double
        L.dfkm_needed.argtypes = [C.c_int, C.c_int, C.c_double]
        L.dfkm_needed.restype = C.c_double
        L.dfkm_hypothesis_counts.argtypes = [C.POINTER(Params), C.c_void_p, C.c_int, C.c_void_p, _I, C.c_int, _I]
        L.dfkm_reprojection_match.argtypes = [C.POINTER(Params), C.c_void_p, C.c_int, C.c_void_p, C.c_int, _I, _I,
                                              _I, _D]
        L.dfkm_reprojection_match.restype = C.c_int
        _lib = L
    return _lib


def _f32(a, shape1=2):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, shape1))


def _ptr(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def hamming(d0, d1) -> np.ndarray:
    """[N0, 2] int32: (train index, distance) per query, (-1, -1) for an empty train set"""
    d0 = np.ascontiguousarray(d0, np.uint8)
    d1 = np.ascontiguousarray(d1, np.uint8)
    assert d0.ndim == 2 and d1.ndim == 2 and d0.shape[1] == d1.shape[1]
    out = np.zeros((d0.shape[0], 2), np.int32)
    lib().dfkm_hamming(d0.ctypes.data, d0.shape[0], d1.ctypes.data, d1.shape[0], d0.shape[1], _ptr(out, C.c_int32))
    return out


def sample(seed: int, h: int, n: int):
    idx = np.zeros(8, np.int32)
    ok = lib().dfkm_sample(seed, h, n, _ptr(idx, C.c_int32))
    return idx if ok else None


def bearings(xy, cam) -> np.ndarray:
    xy = _f32(xy)
    out = np.zeros((xy.shape[0], 3))
    for i in range(xy.shape[0]):
        lib().dfkm_bearing(float(xy[i, 0]), float(xy[i, 1]), cam.fx, cam.fy, cam.u0, cam.v0, _ptr(out[i], C.c_double))
    return out


def eightpt(f0, f1):
    """E (3x3, row-major null vector of the 8 x 9 system f1^T E f0 = 0), or None for a rank-deficient sample"""
    f0 = np.ascontiguousarray(f0, np.float64)
    f1 = np.ascontiguousarray(f1, np.float64)
    e = np.zeros(9)
    ok = lib().dfkm_eightpt(_ptr(f0, C.c_double), _ptr(f1, C.c_double), _ptr(e, C.c_double))
    return e.reshape(3, 3) if ok else None


def model(f0, f1):
    """(R, t) with X1 = R X0 + t, or None for an invalid sample"""
    f0 = np.ascontiguousarray(f0, np.float64)
    f1 = np.ascontiguousarray(f1, np.float64)
    R, t = np.zeros(9), np.zeros(3)
    ok = lib().dfkm_model(_ptr(f0, C.c_double), _ptr(f1, C.c_double), _ptr(R, C.c_double), _ptr(t, C.c_double))
    return (R.reshape(3, 3), t) if ok else None


def score(R, t, f0, f1) -> float:
    R = np.ascontiguousarray(R, np.float64)
    t = np.ascontiguousarray(t, np.float64)
    f0 = np.ascontiguousarray(f0, np.float64)
    f1 = np.ascontiguousarray(f1, np.float64)
    return lib().dfkm_score(_ptr(R, C.c_double), _ptr(t, C.c_double), _ptr(f0, C.c_double), _ptr(f1, C.c_double))


def needed(best: int, n: int, probability: float) -> float:
    return lib().dfkm_needed(best, n, probability)


def params(cam, max_dist=30.0, max_iterations=1000, threshold=float(np.float32(1e-4)), probability=0.99,
           seed=0) -> Params:
    return Params(float(cam.fx), float(cam.fy), float(cam.u0), float(cam.v0), float(threshold), float(probability),
                  float(max_dist), int(max_iterations), int(seed))


def hypothesis_counts(p: Params, kp0, kp1, matches, num: int) -> np.ndarray:
    kp0, kp1 = _f32(kp0), _f32(kp1)
    train = np.ascontiguousarray(np.asarray(matches, np.int32).reshape(-1, 2)[:, 0])
    out = np.zeros(num, np.int32)
    lib().dfkm_hypothesis_counts(C.byref(p), kp0.ctypes.data, kp0.shape[0], kp1.ctypes.data, _ptr(train, C.c_int32),
                                 num, _ptr(out, C.c_int32))
    return out


@dataclass
class MatchResult:
    rows: np.ndarray      # [M, 3] int32: query, train, distance, sorted by (distance, query)
    best: int             # the selected hypothesis, -1 for none
    inliers: int          # its inlier count
    evaluated: int        # hypotheses the adaptive loop evaluated
    scores: np.ndarray    # [N0] float64: every match's score under the selected hypothesis (NaN without one)


def reprojection_match(p: Params, kp0, d0, kp1, d1, matches=None) -> MatchResult:
    """the three steps of one factor: matching (or the given matches), the sequential RANSAC, the distance pruning"""
    kp0, kp1 = _f32(kp0), _f32(kp1)
    m = hamming(d0, d1) if matches is None else np.ascontiguousarray(matches, np.int32).reshape(-1, 2)
    n0 = kp0.shape[0]
    out = np.zeros((max(n0, 1), 3), np.int32)
    stats = np.zeros(3, np.int32)
    scores = np.zeros(max(n0, 1))
    num = lib().dfkm_reprojection_match(C.byref(p), kp0.ctypes.data, n0, kp1.ctypes.data, kp1.shape[0],
                                        _ptr(m, C.c_int32), _ptr(out, C.c_int32), _ptr(stats, C.c_int32),
                                        _ptr(scores, C.c_double))
    return MatchResult(out[:num].copy(), int(stats[0]), int(stats[1]), int(stats[2]), scores[:n0].copy())
